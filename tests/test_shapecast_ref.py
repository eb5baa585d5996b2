"""The numpy restatement of nb_shapecast (oracle/shapecast_ref.py) on the CPU: analytic times of impact (a sphere onto a box face, edge and
corner of axis-aligned and rotated boxes, sphere onto sphere, box onto box face to face, a rotated box pair whose contact only a cross
axis decides, parallel edges, motion parallel to a face inside and outside the slab, max_t stopping short, casts starting in contact,
ties, degenerate casts, masks, ignore_body and sensors); a float64 check of the stated arithmetic's time of impact and normal against a
bisection of the exact overlap predicate along the path, independent of the restatement, on seeded random pairs of every shape
combination; the statement's invariants (a sphere cast of radius 0 is raycast_ref's ray byte for byte, and a cast with max_t = 0 hits at
t = 0 wherever overlap_ref finds its shape in contact); and the nb_shape_cast layout against the header."""
import os
import subprocess
import numpy as np
from nudge_b200 import abi, scenes
from oracle import overlap_ref, raycast_ref, shapecast_ref
from oracle.joints_ref import qrot
from tests.test_raycast_ref import _scene, UNIT, S45, ROOT

NAN, INF = float("nan"), float("inf")
ID = (0.0, 0.0, 0.0, 1.0)


def _c(shape, c, d, max_t=100.0, r=0.0, rot=ID, h=(0.0, 0.0, 0.0), mask=0xffffffff, ignore=abi.RAY_NO_HIT):
    x = np.zeros(1, abi.SHAPE_CAST)
    q = x["shape"]
    q["shape"], q["center"], q["radius"], q["rotation"], q["half_extents"], q["mask"], q["ignore_body"] = shape, c, r, rot, h, mask, ignore
    x["direction"], x["max_t"] = d, max_t
    return x


def sphere(c, r, d, **kw):
    return _c(abi.OVERLAP_SPHERE, c, d, r=r, **kw)


def box(c, h, d, rot=ID, **kw):
    return _c(abi.OVERLAP_BOX, c, d, rot=rot, h=h, **kw)


def _hit(scene, c, flags=0):
    return shapecast_ref.cast(scene, c, flags)[0]


def _is_miss(h):
    return h["collider"] == h["body"] == h["tag"] == abi.RAY_NO_HIT and h.tobytes()[:28] == bytes(28) and h.tobytes()[40:] == bytes(8)


def _rot(q, v):
    return np.array(qrot(tuple(np.float64(x) for x in q), tuple(np.float64(x) for x in v)))


def test_sphere_onto_a_box_face():
    s = _scene([UNIT])
    h = _hit(s, sphere((-5.0, 0.0, 0.0), 0.5, (1.0, 0.0, 0.0)))
    assert h["t"] == 3.5 and tuple(h["position"]) == (-1.5, 0.0, 0.0) and tuple(h["normal"]) == (-1.0, 0.0, 0.0)
    assert (h["collider"], h["body"], h["tag"]) == (0, 1, 100) and h["reserved"].tolist() == [0, 0]


def _rotated_cases(q):
    """(start, direction, radius, t, normal) of a sphere onto the face, the +x+y edge and the +x+y+z corner of the unit box turned by q."""
    cases = [((-5.0, 0.2, 0.1), (1.0, 0.0, 0.0), 0.5, 3.5, (-1.0, 0.0, 0.0)),
             ((5.0, 1.6, 0.0), (-1.0, 0.0, 0.0), 1.0, 3.2, (0.8, 0.6, 0.0)),
             ((5.0, 1.6, 1.6), (-1.0, 0.0, 0.0), 1.0, 4.0 - np.sqrt(0.28), (np.sqrt(0.28), 0.6, 0.6))]
    return [(_rot(q, o), _rot(q, d), r, t, _rot(q, n)) for o, d, r, t, n in cases]


def test_sphere_onto_a_box_edge_and_corner_axis_aligned_and_rotated():
    for q in (ID, (0.0, 0.0, S45, S45), (0.1825742, 0.3651484, 0.5477226, 0.7302967)):
        s = _scene([((0.0, 0.0, 0.0), (1.0, 1.0, 1.0), q)])
        for o, d, r, t, n in _rotated_cases(q):
            h = _hit(s, sphere(tuple(o), r, tuple(d)))
            assert h["collider"] == 0 and abs(h["t"] - t) < 2e-5, (q, o, h["t"], t)
            assert np.abs(h["normal"] - n).max() < 2e-5 and np.abs(h["position"] - (o + h["t"] * d)).max() < 1e-5


def test_sphere_onto_sphere():
    s = _scene(spheres=[((0.0, 0.0, 0.0), 2.0)])
    h = _hit(s, sphere((-5.0, 0.0, 0.0), 1.0, (1.0, 0.0, 0.0)))
    assert h["t"] == 2.0 and tuple(h["normal"]) == (-1.0, 0.0, 0.0) and tuple(h["position"]) == (-3.0, 0.0, 0.0)
    h = _hit(s, sphere((0.0, 10.0, 0.0), 1.0, (0.0, -2.0, 0.0)))   # direction not unit: t in units of its length
    assert h["t"] == 3.5 and tuple(h["normal"]) == (0.0, 1.0, 0.0)
    h = _hit(s, sphere((-5.0, 3.0, 0.0), 1.0, (1.0, 0.0, 0.0)))   # grazing: the centre passes at exactly 2 + 1
    assert h["t"] == 5.0 and tuple(h["normal"]) == (0.0, 1.0, 0.0)
    assert _is_miss(_hit(s, sphere((-5.0, 3.5, 0.0), 1.0, (1.0, 0.0, 0.0))))


def test_box_onto_a_box_face_to_face_at_integer_coordinates():
    s = _scene([UNIT])
    h = _hit(s, box((-5.0, 0.0, 0.0), (1.0, 1.0, 1.0), (1.0, 0.0, 0.0)))
    assert h["t"] == 3.0 and tuple(h["position"]) == (-2.0, 0.0, 0.0) and tuple(h["normal"]) == (-1.0, 0.0, 0.0)
    h = _hit(s, box((0.0, 7.0, 0.0), (2.0, 1.0, 2.0), (0.0, -1.0, 0.0)))
    assert h["t"] == 5.0 and tuple(h["normal"]) == (0.0, 1.0, 0.0)


def test_a_rotated_box_pair_whose_contact_a_cross_axis_decides():
    """overlap_ref's pair: the query turned 45 degrees about z has an edge along z at y = sqrt(2), the collider turned 45 degrees about x one
    along x at y = 3 - sqrt(2).  Moving the query along y, the edges meet at y = 3 - 2 sqrt(2); only cross(u_z, v_x) = y decides that."""
    s8, c8 = float(np.sin(np.pi / 8)), float(np.cos(np.pi / 8))
    rz, rx = (0.0, 0.0, s8, c8), (s8, 0.0, 0.0, c8)
    s = _scene([((0.0, 3.0, 0.0), (1.0, 1.0, 1.0), rx)])
    h = _hit(s, box((0.0, 0.0, 0.0), (1.0, 1.0, 1.0), (0.0, 1.0, 0.0), rot=rz, max_t=1.0))
    assert h["collider"] == 0 and abs(h["t"] - (3.0 - 2.0 * np.sqrt(2.0))) < 1e-5
    assert np.abs(h["normal"] - (0.0, -1.0, 0.0)).max() < 1e-5


def test_parallel_edges_with_zero_cross_axes():
    s = _scene([((5.0, 5.0, 5.0), (1.0, 2.0, 3.0), ID)])
    h = _hit(s, box((5.0, 5.0, 12.0), (1.0, 1.0, 1.0), (0.0, 0.0, -1.0)))
    assert h["t"] == 3.0 and tuple(h["normal"]) == (0.0, 0.0, 1.0)
    h = _hit(s, box((5.5, 4.0, 12.0), (1.0, 1.0, 1.0), (0.0, 0.0, -2.0)))
    assert h["t"] == 1.5 and tuple(h["normal"]) == (0.0, 0.0, 1.0)


def test_motion_parallel_to_a_face_inside_and_outside_the_slab():
    s = _scene([UNIT])
    h = _hit(s, box((-5.0, 1.5, 0.0), (1.0, 0.5, 1.0), (1.0, 0.0, 0.0)))   # b == 0 on y, |a| = 1.5 <= 1.5: touching the slab
    assert h["t"] == 3.0 and tuple(h["normal"]) == (-1.0, 0.0, 0.0)
    assert _is_miss(_hit(s, box((-5.0, 2.0, 0.0), (1.0, 0.5, 1.0), (1.0, 0.0, 0.0))))
    h = _hit(s, sphere((-5.0, 1.25, 0.0), 0.5, (1.0, 0.0, 0.0)))   # over the top edge: the +y face box's slab
    assert h["collider"] == 0 and 3.5 < h["t"] < 4.0 and h["normal"][1] > 0
    assert _is_miss(_hit(s, sphere((-5.0, 1.75, 0.0), 0.5, (1.0, 0.0, 0.0))))


def test_max_t_stops_short():
    s = _scene([UNIT])
    assert _is_miss(_hit(s, sphere((-5.0, 0.0, 0.0), 0.5, (1.0, 0.0, 0.0), max_t=3.4)))
    assert _hit(s, sphere((-5.0, 0.0, 0.0), 0.5, (1.0, 0.0, 0.0), max_t=3.5))["t"] == 3.5
    assert _is_miss(_hit(s, box((-5.0, 0.0, 0.0), (1.0, 1.0, 1.0), (1.0, 0.0, 0.0), max_t=2.9)))
    assert _hit(s, box((-5.0, 0.0, 0.0), (1.0, 1.0, 1.0), (1.0, 0.0, 0.0), max_t=3.0))["t"] == 3.0


def test_a_cast_starting_in_contact_hits_at_t_0_with_a_zero_normal():
    s = _scene([UNIT], [((10.0, 0.0, 0.0), 1.0)])
    for c in (sphere((1.5, 0.0, 0.0), 0.5, (1.0, 0.0, 0.0)), sphere((0.0, 0.0, 0.0), 0.1, (0.0, 1.0, 0.0)),
              box((2.0, 0.0, 0.0), (1.0, 1.0, 1.0), (0.0, 1.0, 0.0)), box((0.5, 0.5, 0.5), (0.1, 0.1, 0.1), (1.0, 0.0, 0.0), rot=(0.0, 0.0, S45, S45))):
        h = _hit(s, c)
        assert h["t"] == 0.0 and h["collider"] == 0 and h.tobytes()[12:28] == bytes(16)
        assert tuple(h["position"]) == tuple(c["shape"]["center"][0])
    h = _hit(s, box((8.5, 0.0, 0.0), (0.5, 0.5, 0.5), (-1.0, 0.0, 0.0)))   # box against the sphere collider
    assert h["t"] == 0.0 and h["collider"] == 1 and tuple(h["normal"]) == (0.0, 0.0, 0.0)


def test_ties_go_to_the_smaller_collider_index():
    s = _scene([UNIT, UNIT], [((0.0, 0.0, 0.0), 1.0)])
    assert _hit(s, sphere((-5.0, 0.0, 0.0), 0.5, (1.0, 0.0, 0.0)))["collider"] == 0
    s = _scene([((0.0, 0.0, 3.0), (1.0, 1.0, 1.0), ID), ((0.0, 0.0, -3.0), (1.0, 1.0, 1.0), ID)], [((0.0, 0.0, 0.0), 1.0)])
    h = _hit(s, box((-5.0, 0.0, 0.0), (1.0, 1.0, 2.0), (1.0, 0.0, 0.0)))   # all three at t = 3
    assert h["t"] == 3.0 and h["collider"] == 0
    s = _scene([((0.0, 0.0, 3.0), (1.0, 1.0, 1.0), ID)], [((0.0, 0.0, -3.0), 1.0)])
    h = _hit(s, sphere((-5.0, 0.0, 0.0), 3.0, (1.0, 0.0, 0.0)))   # box face (t = 1) before the sphere
    assert h["collider"] == 0


def test_degenerate_casts_hit_nothing():
    s = _scene([UNIT], [((0.0, 0.0, 0.0), 1.0)])
    c, d = (-5.0, 0.0, 0.0), (1.0, 0.0, 0.0)
    bad = [_c(2, c, d, r=1.0), sphere((NAN, 0.0, 0.0), 1.0, d), sphere(c, -1.0, d), sphere(c, INF, d), box(c, (1.0, -1.0, 1.0), d),
           box(c, (1.0, 1.0, 1.0), d, rot=(0.0, 0.0, 0.0, 0.0)), box(c, (1.0, 1.0, NAN), d), sphere(c, 1.0, (NAN, 0.0, 0.0)),
           sphere(c, 1.0, (1.0, INF, 0.0)), sphere(c, 1.0, (0.0, 0.0, 0.0)), sphere(c, 1.0, (-0.0, 0.0, -0.0)), sphere(c, 1.0, d, max_t=-1.0),
           sphere(c, 1.0, d, max_t=NAN), sphere(c, 1.0, d, max_t=INF), box(c, (1.0, 1.0, 1.0), d, max_t=-INF)]
    out = shapecast_ref.cast(s, np.concatenate(bad))
    assert all(_is_miss(h) for h in out)
    assert _hit(s, sphere(c, 1.0, d, max_t=0.0, h=(NAN, -1.0, 0.0)))["collider"] == abi.RAY_NO_HIT   # fields a sphere does not read
    assert _hit(s, sphere((-1.5, 0.0, 0.0), 1.0, d, max_t=0.0))["collider"] == 0


def test_masks_ignore_body_and_sensors():
    filt = np.zeros(3, scenes.FILTER); filt["category"] = (0x0002, 0x0004, 0x0002)
    s = _scene([UNIT, ((3.0, 0.0, 0.0), (1.0, 1.0, 1.0), ID)], [((6.0, 0.0, 0.0), 1.0)], filters=filt, sensors=np.array([1, 0, 0], np.uint8))
    c = lambda **kw: sphere((-5.0, 0.0, 0.0), 0.5, (1.0, 0.0, 0.0), **kw)
    assert _hit(s, c())["collider"] == 1                              # the sensor is skipped by default
    assert _hit(s, c(), abi.SHAPECAST_SENSORS)["collider"] == 0
    assert _hit(s, c(mask=0x0002))["collider"] == 2
    assert _is_miss(_hit(s, c(mask=0x0001), abi.SHAPECAST_SENSORS))
    assert _hit(s, c(ignore=2))["collider"] == 2
    assert _hit(s, c(ignore=1), abi.SHAPECAST_SENSORS)["collider"] == 1


# ---- the geometry check: float64, independent of the restatement ----

def _unit_quats(rng, n):
    v = rng.normal(size=(n, 4))
    return v / np.linalg.norm(v, axis=1, keepdims=True)


def _mat(q):
    """Rotation matrices (n, 3, 3) of unit quaternions (x, y, z, w)."""
    x, y, z, w = q.T
    return np.stack([np.stack([1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)], -1),
                     np.stack([2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)], -1),
                     np.stack([2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)], -1)], 1)


def _box_dist(l, h):
    return np.linalg.norm(np.maximum(np.abs(l) - h, 0.0), axis=-1)


def _overlaps(kind, c, U, H, r, p, V, h, rc):
    """The exact overlap predicate in float64, vectorised over pairs (kind: 'ss', 'sb', 'bs', 'bb')."""
    if kind == "ss":
        return np.linalg.norm(c - p, axis=-1) <= r + rc
    if kind == "sb":
        return _box_dist(np.einsum("nji,nj->ni", V, c - p), h) <= r
    if kind == "bs":
        return _box_dist(np.einsum("nji,nj->ni", U, p - c), H) <= rc
    t = p - c
    sep = np.zeros(len(c), bool)
    axes = [U[:, :, i] for i in range(3)] + [V[:, :, j] for j in range(3)] + [np.cross(U[:, :, i], V[:, :, j]) for i in range(3) for j in range(3)]
    for L in axes:
        ra = sum(np.abs(H[:, k] * np.einsum("ni,ni->n", U[:, :, k], L)) for k in range(3))
        rb = sum(np.abs(h[:, k] * np.einsum("ni,ni->n", V[:, :, k], L)) for k in range(3))
        big = np.linalg.norm(L, axis=-1) > 1e-9
        sep |= big & (np.abs(np.einsum("ni,ni->n", t, L)) > ra + rb)
    return ~sep


def _first_contact(kind, c, d, U, H, r, p, V, h, rc, max_t, samples=4000):
    """The smallest t in [0, max_t] at which the shapes overlap (bisection of the float64 predicate), NaN where they never do."""
    at = lambda t: _overlaps(kind, c + t[:, None] * d, U, H, r, p, V, h, rc)
    n = len(c)
    first = np.full(n, np.nan)
    prev = np.zeros(n)
    for s in range(samples + 1):
        t = np.full(n, max_t * s / samples)
        now = np.isnan(first) & at(t)
        first[now] = t[now]
        if s == 0:
            first[now] = 0.0
        else:
            prev[now] = max_t * (s - 1) / samples
    lo, hi = prev.copy(), first.copy()
    todo = ~np.isnan(first) & (first > 0)
    for _ in range(60):
        mid = 0.5 * (lo + hi)
        o = at(np.where(todo, mid, 0.0)) & todo
        hi = np.where(o, mid, hi); lo = np.where(todo & ~o, mid, lo)
    return np.where(todo, hi, first)


def _pairs(kind, rng, n):
    """n seeded pairs whose path passes through the collider (so the contact is not grazing) and n that pass well clear."""
    c = rng.normal(size=(2 * n, 3)) * 3.0
    d = rng.normal(size=(2 * n, 3)); d /= np.linalg.norm(d, axis=1, keepdims=True); d *= rng.uniform(0.5, 2.0, (2 * n, 1))
    qa, qb = _unit_quats(rng, 2 * n), _unit_quats(rng, 2 * n)
    qa[::7] = (0.0, 0.0, 0.0, 1.0); qb[::5] = (0.0, 0.0, 0.0, 1.0)
    H, h = rng.uniform(0.1, 1.0, (2 * n, 3)), rng.uniform(0.1, 1.0, (2 * n, 3))
    r, rc = rng.uniform(0.05, 0.8, 2 * n), rng.uniform(0.05, 0.8, 2 * n)
    off = rng.normal(size=(2 * n, 3)) * 0.15
    side = np.cross(d[n:], rng.normal(size=(n, 3)))   # perpendicular to the path
    off[n:] = side * (6.0 / np.linalg.norm(side, axis=1))[:, None]
    p = c + d * rng.uniform(1.0, 3.0, (2 * n, 1)) + off
    f32 = lambda a: a.astype(np.float32).astype(np.float64)
    return f32(c), f32(d), f32(qa), f32(H), f32(r), f32(p), f32(qb), f32(h), f32(rc)


def _run_pairs(kind, c, d, qa, H, r, p, qb, h, rc, max_t):
    out = np.zeros(len(c), abi.RAY_HIT)
    for k in range(len(c)):
        boxes = [(tuple(p[k]), tuple(h[k]), tuple(qb[k]))] if kind[1] == "b" else []
        spheres = [] if boxes else [(tuple(p[k]), float(rc[k]))]
        s = _scene(boxes, spheres)
        cs = sphere(tuple(c[k]), float(r[k]), tuple(d[k]), max_t=max_t) if kind[0] == "s" else \
            box(tuple(c[k]), tuple(H[k]), tuple(d[k]), rot=tuple(qa[k]), max_t=max_t)
        out[k] = shapecast_ref.cast(s, cs)[0]
    return out


def _normal64(kind, c, U, H, r, p, V, h, rc):
    """The float64 contact normal (from the collider towards the cast shape) at a touching configuration, for a sphere on either side."""
    if kind == "ss":
        v = c - p
    elif kind == "sb":
        l = np.einsum("nji,nj->ni", V, c - p)
        v = np.einsum("nij,nj->ni", V, l - np.clip(l, -h, h))
    else:
        l = np.einsum("nji,nj->ni", U, p - c)
        v = -np.einsum("nij,nj->ni", U, l - np.clip(l, -H, H))
    return v / np.linalg.norm(v, axis=1, keepdims=True)


def test_the_stated_arithmetic_finds_the_geometric_time_of_impact():
    rng = np.random.default_rng(77)
    max_t = 4.0
    for kind in ("ss", "sb", "bs", "bb"):
        n = 600
        c, d, qa, H, r, p, qb, h, rc = _pairs(kind, rng, n)
        U, V = _mat(qa), _mat(qb)
        got = _run_pairs(kind, c, d, qa, H, r, p, qb, h, rc, max_t)
        want = _first_contact(kind, c, d, U, H, r, p, V, h, rc, max_t)
        hit = got["collider"] != abi.RAY_NO_HIT
        assert (hit == ~np.isnan(want)).all(), (kind, np.nonzero(hit != ~np.isnan(want))[0][:5])
        assert hit[:n].mean() > 0.9 and not hit[n:].any(), kind
        t = got["t"].astype(np.float64)
        err = np.abs(t[hit] - want[hit]) / np.maximum(1.0, want[hit])
        assert err.max() < 1e-4, (kind, err.max())
        at = hit & (t > 0)
        if kind == "bb":   # every contact: the normal's plane supports both boxes at the hit, with a zero gap
            cc = c[at] + t[at, None] * d[at]
            nn = got["normal"][at].astype(np.float64)
            Ua, Va = U[at], V[at]
            ra = sum(np.abs(H[at, k] * np.einsum("ni,ni->n", Ua[:, :, k], nn)) for k in range(3))
            rb = sum(np.abs(h[at, k] * np.einsum("ni,ni->n", Va[:, :, k], nn)) for k in range(3))
            gap = np.einsum("ni,ni->n", cc - p[at], nn) - (ra + rb)
            assert np.abs(np.linalg.norm(nn, axis=1) - 1).max() < 1e-5 and np.abs(gap).max() < 1e-3, np.abs(gap).max()
        else:              # a sphere on either side: the contact normal is unique
            cc = c[at] + t[at, None] * d[at]
            nn = _normal64(kind, cc, U[at], H[at], r[at], p[at], V[at], h[at], rc[at])
            assert np.abs(got["normal"][at] - nn).max() < 1e-3, (kind, np.abs(got["normal"][at] - nn).max())


# ---- the invariants of the statement ----

def _scene_of(rng, nb=40, ns=40):
    boxes = [(tuple(rng.uniform(-6, 6, 3)), tuple(rng.uniform(0.2, 1.2, 3)), tuple(_unit_quats(rng, 1)[0])) for _ in range(nb)]
    spheres = [(tuple(rng.uniform(-6, 6, 3)), float(rng.uniform(0.2, 1.0))) for _ in range(ns)]
    return _scene(boxes, spheres)


def test_a_sphere_cast_of_radius_0_is_the_ray_byte_for_byte():
    for seed in range(4):
        rng = np.random.default_rng(100 + seed)
        s = _scene_of(rng)
        n = 300
        rays = np.zeros(n, abi.RAY)
        rays["origin"] = rng.uniform(-9, 9, (n, 3)); rays["direction"] = rng.normal(size=(n, 3)) * rng.uniform(0.1, 3.0, (n, 1))
        rays["max_t"] = rng.uniform(0, 20, n); rays["mask"] = 0xffffffff; rays["ignore_body"] = abi.RAY_NO_HIT
        rays["direction"][::9, 1] = 0.0; rays["max_t"][::11] = 0.0; rays["direction"][::13] = (0.0, -1.0, 0.0)
        casts = np.zeros(n, abi.SHAPE_CAST)
        casts["shape"]["shape"] = abi.OVERLAP_SPHERE; casts["shape"]["center"] = rays["origin"]; casts["shape"]["mask"] = 0xffffffff
        casts["shape"]["ignore_body"] = abi.RAY_NO_HIT; casts["direction"] = rays["direction"]; casts["max_t"] = rays["max_t"]
        want = raycast_ref.cast(s, rays)
        got = shapecast_ref.cast(s, casts)
        assert got.tobytes() == want.tobytes()
        assert (want["collider"] != abi.RAY_NO_HIT).sum() >= 25


def test_a_cast_with_max_t_0_hits_where_the_overlap_query_finds_contact():
    rng = np.random.default_rng(55)
    s = _scene_of(rng)
    n = 400
    q = np.zeros(n, abi.OVERLAP_QUERY)
    q["shape"] = rng.integers(0, 2, n); q["center"] = rng.uniform(-7, 7, (n, 3)); q["radius"] = rng.uniform(0, 1.5, n)
    q["rotation"] = _unit_quats(rng, n); q["half_extents"] = rng.uniform(0.1, 1.5, (n, 3)); q["mask"] = 0xffffffff; q["ignore_body"] = abi.RAY_NO_HIT
    casts = np.zeros(n, abi.SHAPE_CAST)
    casts["shape"] = q; casts["direction"] = rng.normal(size=(n, 3)); casts["max_t"] = 0.0
    off, hits = overlap_ref.query(s, q)
    got = shapecast_ref.cast(s, casts)
    touching = 0
    for k in range(n):
        mine = hits["collider"][off[k]:off[k + 1]]
        if len(mine):
            touching += 1
            assert got["t"][k] == 0.0 and got["collider"][k] <= mine.min() and got.tobytes()[48 * k + 12:48 * k + 28] == bytes(16)
    assert touching > n // 4


def test_shape_cast_layout_matches_the_header(tmp_path):
    dt = abi.SHAPE_CAST
    src = tmp_path / "layout.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "nudge_b200.h"\nint main(void) {\n' +
                   "".join('printf("%%zu\\n", offsetof(nb_shape_cast, %s));\n' % k for k in dt.names) +
                   'printf("%zu\\n", offsetof(nb_shape_cast, shape.mask)); printf("%zu\\n", sizeof(nb_shape_cast));'
                   ' printf("%d\\n", (int)NB_SHAPECAST_SENSORS); return 0; }\n')
    exe = tmp_path / "layout"
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), "-o", str(exe), str(src)])
    out = [int(x) for x in subprocess.check_output([str(exe)]).split()]
    assert out[:len(dt.names)] == [dt.fields[k][1] for k in dt.names]
    assert out[len(dt.names):] == [abi.OVERLAP_QUERY.fields["mask"][1], dt.itemsize, abi.SHAPECAST_SENSORS]
    assert dt.itemsize == 80
