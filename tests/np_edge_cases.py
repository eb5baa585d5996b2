"""Edge-case geometry for the narrowphase (box-box, box-sphere, sphere-sphere), in plain numpy.

Every scene is a set of isolated clusters: one case per cluster, far enough from every other cluster that no two clusters pair in
the broadphase.  Each cluster records its family and case id, so a failing contact can be traced to the geometry that made it.
Clusters are laid out in the x-z plane (y = 0), so offsets along y are exact for every cluster; cases that need tiny coordinates
sit alone at the origin of their own scene.  The box and sphere lists are shuffled by cluster, so that neighbouring pairs in the
narrowphase's lists are of different kinds (face, edge, no contact; box-box, box-sphere, sphere-sphere).

tests/golden/make_np_edge_golden.py records what the unmodified reference computes on these scenes into
tests/golden/np_edge_cases.npz; tests/test_np_edges_oracle.py (CPU) and tests/test_gpu_np_edges.py (GPU) compare against it."""
import hashlib
import numpy as np
from nudge_b200 import scenes as S

f32 = np.float32
SPACING = 32.0          # lattice pitch of the ordinary clusters; their colliders stay within SMALL of the cluster centre
SMALL = 12.0
ID = (0.0, 0.0, 0.0, 1.0)


def qaxis(axis, angle):
    """Axis-angle quaternion, computed in float64 and rounded to float32 (what a user would upload)."""
    a = np.asarray(axis, np.float64); a = a / np.linalg.norm(a)
    return tuple(np.append(a * np.sin(angle / 2), np.cos(angle / 2)).astype(f32))


def qmul(a, b):
    """Hamilton product a*b (rotation b first), float64."""
    ax, ay, az, aw = np.asarray(a, np.float64); bx, by, bz, bw = np.asarray(b, np.float64)
    return (aw*bx + ax*bw + ay*bz - az*by, aw*by - ax*bz + ay*bw + az*bx, aw*bz + ax*by - ay*bx + az*bw, aw*bw - ax*bx - ay*by - az*bz)


def qrot(q, v):
    x, y, z, w = np.asarray(q, np.float64)
    u = np.array([x, y, z]); v = np.asarray(v, np.float64)
    t = 2.0 * np.cross(u, v)
    return v + w * t + np.cross(u, t)


def box(size, pos=(0, 0, 0), rot=ID, static=False):
    return dict(shape="box", size=tuple(size), pos=tuple(pos), rot=tuple(rot), static=static)


def sphere(radius, pos=(0, 0, 0), static=False):
    return dict(shape="sphere", radius=radius, pos=tuple(pos), rot=ID, static=static)


def case(family, cid, colliders, touch, origin=False, tag_order=None, **meta):
    """touch: True (must make contacts), False (must not), or an exact contact count.  origin: the case needs exact tiny coordinates
    and gets a scene of its own, centred at the origin.  tag_order: 'first_higher' / 'first_lower' fixes which collider has the higher tag."""
    return dict(family=family, case=cid, colliders=colliders, touch=touch, origin=origin, tag_order=tag_order, meta=meta)


def rotated(cols, q):
    """The whole cluster rotated by q about its centre (float64, rounded to float32 once)."""
    out = []
    for c in cols:
        c = dict(c)
        c["pos"] = tuple(qrot(q, c["pos"]))
        c["rot"] = tuple(np.asarray(qmul(q, c["rot"]), np.float64))
        out.append(c)
    return out


# ---------------- float32 restatement of the face test (nudge.cpp:1195-1410), used only to place the exact-zero grazing case --------------
def _face_p32(sa, pa, qa, sb, pb, qb):
    sa, pa, qa, sb, pb, qb = (np.asarray(v, f32) for v in (sa, pa, qa, sb, pb, qb))
    one = f32(1)
    t = np.cross(qb[:3], qa[:3]).astype(f32)
    r = (qa[:3] * qb[3] - qb[:3] * qa[3] - t).astype(f32)
    rs = f32(qa[0]*qb[0] + qa[1]*qb[1] + qa[2]*qb[2] + qa[3]*qb[3])
    k = (r + r).astype(f32)
    xx, yy, zz, xy, xz, yz = k[0]*r[0], k[1]*r[1], k[2]*r[2], k[0]*r[1], k[0]*r[2], k[1]*r[2]
    sx, sy, sz = k[0]*rs, k[1]*rs, k[2]*rs
    m = np.abs(np.array([one - yy - zz, xy + sz, xz - sy, xy - sz, one - xx - zz, yz + sx, xz + sy, yz - sx, one - xx - yy], f32)).reshape(3, 3)
    p_a = np.array([sb[j] + m[0, j]*sa[0] + m[1, j]*sa[1] + m[2, j]*sa[2] for j in range(3)], f32)
    p_b = np.array([sa[i] + m[i, 0]*sb[0] + m[i, 1]*sb[1] + m[i, 2]*sb[2] for i in range(3)], f32)
    d = (pa - pb).astype(f32)

    def cross(a, b):
        return np.array([a[1]*b[2] - a[2]*b[1], a[2]*b[0] - a[0]*b[2], a[0]*b[1] - a[1]*b[0]], f32)
    t = cross(qb[:3], d); t = t + t; u = cross(qb[:3], t)
    p_a = p_a - np.abs(u + d - qb[3] * t)
    t = cross(d, qa[:3]); t = t + t; u = cross(qa[:3], t)
    p_b = p_b - np.abs(u - d - qa[3] * t)
    return min(p_a.min(), p_b.min())


def _grazing_zero():
    """Two unit boxes sharing a rotation q that is not exact in float32, b above a along a's y axis, nudged by whole ulps in y until
    the face test's penetration is exactly 0 whichever box is first (so `p > 0` must reject) while the AABBs still overlap."""
    q = qaxis((1.0, 0.0, 1.0), 0.3)
    s = (1.0, 1.0, 1.0)
    up = qrot(q, (0.0, 2.0, 0.0)).astype(f32)
    ext = np.abs(np.array([qrot(q, e) for e in np.eye(3)])).sum(0)   # AABB half extents of a unit box rotated by q
    for k in range(-64, 65):
        pb = up.copy()
        for _ in range(abs(k)):
            pb[1] = np.nextafter(pb[1], f32(np.inf) if k > 0 else f32(-np.inf))
        if _face_p32(s, (0, 0, 0), q, s, pb, q) == 0 and _face_p32(s, pb, q, s, (0, 0, 0), q) == 0 and (np.abs(pb) < 2 * ext).all():
            return [box(s, (0, 0, 0), q), box(s, tuple(pb), q)]
    raise AssertionError("no exact-zero grazing position found")


# ---------------- the families ----------------
Y90 = (0.0, 0.70710677, 0.0, 0.70710677)     # 90 degrees about y, as float32 rounds it
X180 = (1.0, 0.0, 0.0, 0.0)                  # exact
Y180 = (0.0, 1.0, 0.0, 0.0)
NEG_ID = (0.0, 0.0, 0.0, -1.0)               # the identity as -q
Z45 = qaxis((0, 0, 1), np.pi / 4)
X45 = qaxis((1, 0, 0), np.pi / 4)
TILT = qaxis((1.0, 2.0, 3.0), 0.7)           # a generic rotation for whole clusters
# b's rotation and offset (a = (1, 0.5, 1) at the centre, b = (bx, 0.5, bz) rotated about y, then tilted about x by `tilt`) for
# face-face manifolds of each size; found by sweeping the parameters through the reference
MANIFOLDS = {
    5: (0.65, 1.1, 0.18, 0.25, 0.9, -0.83, 0.0),
    6: (0.95, 0.77, 0.25, -0.03, 0.9, 0.78, 0.0),
    7: (0.94, 0.81, 0.66, 0.06, 0.9, 0.63, 0.0),
}


def box_box_cases():
    c = []
    F = "box-box"
    u = (1.0, 1.0, 1.0)
    c.append(case(F + " face-face equal", 0, [box(u), box(u, (0, 1.75, 0))], 8))
    c.append(case(F + " face-face equal", 1, [box(u), box(u, (0.5, -1.75, 0.25))], True))
    c.append(case(F + " face-face unequal", 0, [box((2, 1, 2)), box((0.5, 0.5, 0.5), (0, 1.375, 0))], 4))
    c.append(case(F + " face-face unequal", 1, [box((0.5, 0.5, 0.5)), box((2, 1, 2), (0, -1.375, 0))], 4))
    c.append(case(F + " face-face unequal", 2, [box((1, 0.5, 1)), box((1, 0.5, 0.5), (0, 0.875, 0.5))], True))
    c.append(case(F + " face-face unequal", 3, [box((1, 1, 1)), box((1, 1, 1), (0.5, 0.5, 1.75))], True))
    c.append(case(F + " coincident centres", 0, [box(u), box(u)], True))
    c.append(case(F + " coincident centres", 1, [box((1, 0.5, 0.25)), box((0.25, 1, 0.5), (0, 0, 0), Z45)], True))
    for k, (qa, qb) in enumerate([(ID, Y90), (ID, X180), (ID, NEG_ID), (Y90, tuple(-np.asarray(Y90))), (X180, Y180), (NEG_ID, Y90)]):
        c.append(case(F + " exact quaternions", k, [box((1, 0.5, 0.75), (0, 0, 0), qa), box((0.75, 0.5, 1), (0, 0.9375, 0), qb)], True))
    c.append(case(F + " exact quaternions", 6, [box((1, 0.5, 0.75), (0, 0, 0), X180), box((1, 0.5, 0.75), (0.25, 0.9375, 0), tuple(-np.asarray(X180)))], True))
    h = np.sqrt(2.0)
    c.append(case(F + " edge-edge", 0, [box(u, (0, 0, 0), Z45), box(u, (0, 2 * h - 0.05, 0), X45)], True))      # crossing at right angles
    c.append(case(F + " edge-edge", 1, [box(u, (0, 0, 0), Z45), box(u, (0, 2 * h - 0.05, 0), Z45)], True))      # exactly parallel
    near = tuple(np.asarray(qmul(qaxis((0, 1, 0), 1e-7), Z45), np.float64))
    c.append(case(F + " edge-edge", 2, [box(u, (0, 0, 0), Z45), box(u, (0, 2 * h - 0.05, 0), near)], True))     # ~1e-7 rad apart
    c.append(case(F + " edge-edge", 3, rotated([box(u, (0, 0, 0), Z45), box(u, (0, 2 * h - 0.05, 0), X45)], TILT), True))
    c.append(case(F + " edge-edge", 4, [box((1, 0.5, 2), (0, 0, 0), Z45), box((2, 0.5, 1), (0.1, 0.5 * h + 0.5 * h - 0.02, 0), X45)], True))
    corner = tuple(np.asarray(qmul(qaxis((0, 0, 1), np.arctan(1 / h)), qaxis((1, 0, 0), np.pi / 4)), np.float64))
    c.append(case(F + " vertex into face", 0, [box((2, 0.5, 2)), box(u, (0, 0.5 + np.sqrt(3) - 0.05, 0), corner)], True))
    c.append(case(F + " vertex into face", 1, rotated([box((2, 0.5, 2)), box(u, (0.3, 0.5 + np.sqrt(3) - 0.01, -0.2), corner)], TILT), True))
    c.append(case(F + " survives faces, no contact", 0, rotated([box(u, (0, 0, 0), Z45), box(u, (0, 2 * h + 0.05, 0), X45)], TILT), False))
    c.append(case(F + " survives faces, no contact", 1, rotated([box(u, (0, 0, 0), Z45), box(u, (0.2, 2 * h + 0.02, 0.1), X45)], TILT), False))
    c.append(case(F + " manifold", 1, [box(u, (0, 0, 0), Z45), box(u, (0, 2 * h - 0.05, 0), X45)], 1))
    c.append(case(F + " manifold", 8, [box(u), box(u, (0, 1.9375, 0))], 8))
    for n, (bx, bz, ang, ox, oy, oz, tilt) in sorted(MANIFOLDS.items()):
        qb = tuple(np.asarray(qmul(qaxis((1, 0, 0), tilt) if tilt else ID, qaxis((0, 1, 0), ang)), np.float64))
        c.append(case(F + " manifold", n, [box((1, 0.5, 1)), box((bx, 0.5, bz), (ox, oy, oz), qb)], n))
    eps = float(np.spacing(f32(2.0)))   # one ulp of 2: the face test's penetration is computed as 2 - |delta|
    for k, ulps in enumerate((1, 3)):
        c.append(case(F + " grazing", k, [box(u), box(u, (0, 2.0 - ulps * eps / 2, 0))], True, ulps=ulps))
    c.append(case(F + " grazing", 2, _grazing_zero(), False, origin=True))
    c.append(case(F + " extreme aspect", 0, [box((1e-3, 1, 1e3), (0, 0, 0)), box((1e-3, 1, 1e3), (1.9e-3, 0, 0))], True))
    c.append(case(F + " extreme aspect", 1, [box((1e3, 1e-3, 1)), box((1, 1, 1e-3), (0, 0.99, 0), Z45)], True))
    c.append(case(F + " large scale", 0, [box((1e4, 1e4, 1e4)), box((1e4, 1e4, 1e4), (0, 1.9e4, 0))], True))
    c.append(case(F + " large scale", 1, [box((1e4, 1e4, 1e4), (0, 0, 0), Z45), box((1e4, 1e4, 1e4), (0, 2e4 * h - 400, 0), X45)], True))
    # The reference's face clipper stops reporting contacts between half sizes 2^-63 and 2^-64, where the squares of sizes become
    # subnormal, and its edge-edge test between 2^-9 and 2^-10: each scale is recorded on both sides of that edge.
    for k, (p, touch) in enumerate(((-63, True), (-64, False), (-140, False))):
        s = 2.0 ** p
        c.append(case(F + " tiny scale, face", k, [box((s, s, s)), box((s, s, s), (0.5 * s, 1.875 * s, 0.25 * s))], touch, origin=True))
    for k, (p, touch) in enumerate(((-9, True), (-10, False))):
        s = 2.0 ** p
        c.append(case(F + " tiny scale, edge", k, [box((s, s, s), (0, 0, 0), Z45), box((s, s, s), (0, 2.75 * s, 0), X45)], touch, origin=True))
    for k, scale in enumerate((1.001, 0.999)):
        c.append(case(F + " unnormalised quaternion", k, [box(u, (0, 0, 0), tuple(np.asarray(Z45, np.float64) * scale)),
                                                         box(u, (0.1, 2 * h - 0.05, 0), tuple(np.asarray(X45, np.float64) * scale))], True))
        c.append(case(F + " unnormalised quaternion", 2 + k, [box(u), box(u, (0.25, 1.9, 0), tuple(np.asarray(Z45, np.float64) * scale))], True))
    return c


def main_cpp_cases():
    """The five two-box configurations of the reference's own tests (tests/golden/make_golden.py), first orientation of each."""
    from tests.golden.make_golden import cases as golden_cases
    seen, out = set(), []
    for g in golden_cases():
        if g["family"] in seen:
            continue
        seen.add(g["family"])
        cols = []
        for i in range(2):
            static = g["cbody"][i] == 0
            pos, rot = np.asarray(g["cpos"][i], np.float64), np.asarray(g["crot"][i], np.float64)
            if not static and "bpos" in g:
                pos, rot = np.asarray(g["bpos"], np.float64), np.asarray(g["brot"], np.float64)
            cols.append(box(g["size"][i], pos, rot, static=static))
        out.append(case("box-box tests/main.cpp", int(g["family"]), cols, int(g["expect"])))
    return out


def box_sphere_cases():
    c = []
    F = "box-sphere"
    s = (1.0, 0.75, 0.5)   # unequal half sizes: every face distance is distinct
    r = 0.25
    for k, off in enumerate([(0.875, 0, 0), (-0.875, 0, 0), (0, 0.625, 0), (0, -0.625, 0), (0, 0, 0.375), (0, 0, -0.375)]):
        c.append(case(F + " inside, nearest face", k, [box(s), sphere(r, off)], True))
    for k, off in enumerate([(0.75, 0.5, 0), (-0.75, 0.5, 0.1), (0.75, 0, 0.25), (0.1, -0.5, 0.25)]):
        c.append(case(F + " equidistant from two faces", k, [box(s), sphere(r, off)], True))
    for k, off in enumerate([(0.75, 0.5, 0.25), (-0.75, -0.5, -0.25), (0, 0, 0)]):
        c.append(case(F + " equidistant from three faces", k, [box((1, 1, 1) if k == 2 else s), sphere(r, off)], True))
    for k, off in enumerate([(1.0, 0.25, 0), (-1.0, 0.75, 0), (0, 0.75, 0.5), (1.0, 0.75, 0.5)]):
        c.append(case(F + " centre on a face plane", k, [box(s), sphere(r, off)], True))
    w = 1.25
    c.append(case(F + " dx == size + r", 0, [box(s), sphere(r, (w, 0, 0))], False))
    c.append(case(F + " dx == size + r", 1, [box(s), sphere(r, (0, -1.0, 0))], False))
    c.append(case(F + " dx == size + r", 2, [box(s), sphere(r, (0, float(np.nextafter(f32(1.0), f32(0))), 0))], True))
    # b's offset in the rotated box's frame rounds to exactly (w, 0, 0) while the AABBs overlap (an unrotated box's AABB would
    # only touch the sphere's, and the broadphase would drop the pair): found by stepping the position in ulps
    c.append(case(F + " dx == size + r", 3, [box(s, (0, 0, 0), Z45), sphere(r, (0.8838834762573242, 0.8838834166526794, 0.0))], False, origin=True))
    c.append(case(F + " edge region", 0, [box(s), sphere(r, (1.125, 0.875, 0.1))], True))
    c.append(case(F + " edge region", 1, [box(s), sphere(r, (1.2, 0.95, 0))], False))     # inside the slab test, outside the radius
    c.append(case(F + " edge region", 2, [box(s), sphere(0.3125, (-1.1875, 1.0, 0))], True))   # l2 == r*r == 25/256 exactly
    c.append(case(F + " corner region", 0, [box(s), sphere(r, (1.0625, 0.8125, 0.5625))], True))
    c.append(case(F + " corner region", 1, [box(s), sphere(r, (-1.2, 0.95, -0.7))], False))
    c.append(case(F + " sphere larger than box", 0, [box((0.25, 0.25, 0.25)), sphere(2.0, (0, 2.125, 0))], True))
    c.append(case(F + " sphere larger than box", 1, [box((0.25, 0.25, 0.25)), sphere(2.0, (0.1, 0.2, 0))], True))
    c.append(case(F + " sphere larger than box", 2, [box((0.25, 0.25, 0.25)), sphere(2.0, (1.5, 1.5, 0.5))], True))
    for k, off in enumerate([(0, 0.9, 0), (1.0, 0.85, 0.3), (0.3, 0.2, 0.1)]):
        c.append(case(F + " rotated box", k, rotated([box(s), sphere(r, off)], TILT), True))
    c.append(case(F + " rotated box", 3, [box(s, (0, 0, 0), Y90), sphere(r, (0, 0, 1.125))], True))
    t = 2.0 ** -100
    c.append(case(F + " corner l2 underflows", 0, [box((t, t, t)), sphere(2.0 ** -110, (t + 2.0 ** -120, t + 2.0 ** -120, t + 2.0 ** -120))], True, origin=True,
                  nan=True))   # l2 == 0: the normal is infinite and the contact position NaN
    t = 2.0 ** -127
    c.append(case(F + " subnormal", 0, [box((t, 0.75 * t, 0.5 * t)), sphere(2.0 ** -129, (t + 2.0 ** -131, 0, 0))], True, origin=True))
    return c


def _l2_targets():
    """Sphere-centre offsets (a, y, 0) whose float32 l2 = (a*a + y*y) + 0 is 1e-4f and its neighbours one ulp below and above.  a is a
    multiple of 2^-14, so that it stays exact next to any lattice centre; y is free, since every cluster centre has y = 0."""
    lim = f32(1e-4)
    want = {"l2 one ulp below 1e-4f": np.nextafter(lim, f32(0)), "l2 == 1e-4f": lim, "l2 one ulp above 1e-4f": np.nextafter(lim, f32(1))}
    found = {}
    for name, target in want.items():
        for k in range(1, 160):
            a = f32(k * 2.0 ** -14)
            aa = f32(a * a)
            y0 = f32(np.sqrt(np.float64(target) - np.float64(aa)))
            for d in range(-4, 5):
                y = y0
                for _ in range(abs(d)):
                    y = np.nextafter(y, f32(1) if d > 0 else f32(0))
                if f32(f32(aa + f32(y * y)) + f32(0)) == target:
                    found[name] = (float(a), float(y), 0.0)
                    break
            if name in found:
                break
    assert len(found) == 3, found
    return found


def sphere_sphere_cases():
    c = []
    F = "sphere-sphere"
    c.append(case(F + " concentric", 0, [sphere(0.5), sphere(0.75)], True))
    c.append(case(F + " concentric", 1, [sphere(0.5), sphere(0.5, (0, 2.0 ** -20, 0))], True))
    for k, (name, off) in enumerate(sorted(_l2_targets().items())):
        c.append(case(F + " " + name, 0, [sphere(0.5), sphere(0.5, off)], True))
    c.append(case(F + " exactly touching", 0, [sphere(0.25), sphere(0.375, (0.375, 0.5, 0))], True))       # l2 == r*r == 25/64
    c.append(case(F + " exactly touching", 1, [sphere(0.25), sphere(0.375, (0.375, 0.5 + 2.0 ** -20, 0))], False))
    c.append(case(F + " very unequal radii", 0, [sphere(1e-3), sphere(10.0, (0, 10.0005, 0))], True))
    c.append(case(F + " very unequal radii", 1, [sphere(10.0), sphere(1e-3, (3.0, -10.0005, 4.0))], False))
    c.append(case(F + " very unequal radii", 2, [sphere(10.0), sphere(1e-3, (0, 9.9995, 0))], True))
    c.append(case(F + " subnormal", 0, [sphere(2.0 ** -130), sphere(2.0 ** -130, (0, 2.0 ** -131, 2.0 ** -131))], True, origin=True))
    return c


def tag_body_cases():
    c = []
    F = "tags and bodies"
    u = (1.0, 1.0, 1.0)
    k = 0
    for order in ("first_higher", "first_lower"):
        for static in (None, 0, 1):
            cols = [box(u, static=static == 0), box(u, (0.25, 1.875, 0), static=static == 1)]
            c.append(case(F + " box-box", k, cols, True, tag_order=order)); k += 1
            cols = [box(u, static=static == 0), sphere(0.5, (0.25, 1.375, 0), static=static == 1)]
            c.append(case(F + " box-sphere", k, cols, True, tag_order=order)); k += 1
            cols = [sphere(0.5, static=static == 0), sphere(0.75, (0.25, 1.125, 0), static=static == 1)]
            c.append(case(F + " sphere-sphere", k, cols, True, tag_order=order)); k += 1
    return c


def tail_kinds():
    """Box-box cases that all survive the face test, cycled through by the tail scenes: face, edge, face-then-nothing, vertex."""
    h = np.sqrt(2.0)
    u = (1.0, 1.0, 1.0)
    return [[box(u), box(u, (0.25, 1.875, 0))],
            [box(u, (0, 0, 0), Z45), box(u, (0, 2 * h - 0.05, 0), X45)],
            rotated([box(u, (0, 0, 0), Z45), box(u, (0, 2 * h + 0.05, 0), X45)], TILT),
            [box((1, 0.5, 0.25)), box((0.5, 0.5, 0.5), (0.75, 0.875, 0), Z45)]]


# ---------------- scene assembly ----------------
class EdgeScene:
    """scene: nudge_b200.scenes.Scene; clusters: list of cases; col_cluster[i]: the cluster of collider i (boxes, then spheres)."""

    def __init__(self, name, scene, clusters, col_cluster):
        self.name, self.scene, self.clusters, self.col_cluster = name, scene, clusters, col_cluster

    @property
    def nan_blind(self):
        """True if a case makes NaN contacts on purpose: the solver stages that follow are then compared with NaN == NaN
        (parity_util.nan_canonical), since their NaNs' signs depend on operand order."""
        return any(c["meta"].get("nan") for c in self.clusters)

    def cluster_of_tag(self):
        t = np.concatenate([self.scene.box_tags, self.scene.sphere_tags]).astype(np.int64)
        out = np.full(t.max() + 1 if len(t) else 1, -1, np.int64)
        out[t] = self.col_cluster
        return out

    def describe(self, cluster):
        c = self.clusters[cluster]
        return "%s case %d" % (c["family"], c["case"])

    def input_digest(self):
        h = hashlib.sha256()
        s = self.scene
        for a in (s.transforms, s.properties, s.momentum, s.idle, s.box_tags, s.box_data, s.box_transforms, s.sphere_tags, s.sphere_data, s.sphere_transforms):
            h.update(np.ascontiguousarray(a).view(np.uint8).tobytes())
        return np.frombuffer(h.digest()[:8], np.uint8)


def _extent(c):
    e = 0.0
    for col in c["colliders"]:
        half = np.linalg.norm(col["size"]) if col["shape"] == "box" else col["radius"]
        e = max(e, np.linalg.norm(col["pos"]) + half)
    return e


def assemble(name, clusters, seed):
    """Places the clusters (origin case at the origin, ordinary ones on an x-z lattice, large ones further out along -z), shuffles the
    box and sphere lists by cluster, assigns tags and bodies.  Dynamic bodies get unit inverse mass and inertia, whatever their size."""
    rng = np.random.default_rng(seed)
    n = len(clusters)
    centre = np.zeros((n, 3), np.float64)
    small = [i for i, c in enumerate(clusters) if not c["origin"] and _extent(c) <= SMALL]
    big = [i for i, c in enumerate(clusters) if not c["origin"] and _extent(c) > SMALL]
    side = int(np.ceil(np.sqrt(len(small) + 1)))
    slots = [(i, k) for i in range(side) for k in range(side)]
    slots = [s for s in slots if s != (side // 2, side // 2)][:len(small)]   # the lattice's centre is the origin: kept free
    for j, (i, k) in zip(small, slots):
        centre[j] = ((i - side // 2) * SPACING, 0.0, (k - side // 2) * SPACING)
    z = -(side // 2 + 1) * SPACING
    for j in big:
        e = _extent(clusters[j])
        grain = 2.0 ** np.ceil(np.log2(e))     # centres on a power-of-two grain keep the offsets exact
        z = np.floor((z - e - SPACING) / grain) * grain
        centre[j] = (0.0, 0.0, z)
        z -= e
    assert sum(c["origin"] for c in clusters) <= 1

    order = rng.permutation(n)
    boxes = [(j, col) for j in order for col in clusters[j]["colliders"] if col["shape"] == "box"]
    spheres = [(j, col) for j in order for col in clusters[j]["colliders"] if col["shape"] == "sphere"]
    allc = boxes + spheres
    n_dyn = sum(1 for _, col in allc if not col["static"])
    s = S.Scene(1 + n_dyn, len(boxes), len(spheres))
    s.name = name
    s.iterations = 4
    tags = rng.permutation(len(allc)).astype(np.uint32)
    col_cluster = np.array([j for j, _ in allc], np.int64)
    for j, c in enumerate(clusters):   # fix which collider of the cluster carries the higher tag
        if c["tag_order"]:
            idx = [i for i in range(len(allc)) if col_cluster[i] == j]
            first = min(idx, key=lambda i: allc[i][1] is not c["colliders"][0])
            other = [i for i in idx if i != first][0]
            hi, lo = max(tags[first], tags[other]), min(tags[first], tags[other])
            tags[first], tags[other] = (hi, lo) if c["tag_order"] == "first_higher" else (lo, hi)
    body = 1
    nb = len(boxes)
    for i, (j, col) in enumerate(allc):
        pos = (centre[j] + np.asarray(col["pos"], np.float64)).astype(f32)
        rot = np.asarray(col["rot"], np.float64).astype(f32)
        xf = s.box_transforms if i < nb else s.sphere_transforms
        k = i if i < nb else i - nb
        if col["static"]:
            xf["position"][k] = pos; xf["rotation"][k] = rot; xf["body"][k] = 0
        else:
            xf["body"][k] = body
            s.transforms["position"][body] = pos; s.transforms["rotation"][body] = rot
            s.properties["mass_inverse"][body] = 1.0; s.properties["inertia_inverse"][body] = 1.0
            body += 1
        if i < nb:
            s.box_data["size"][k] = col["size"]; s.box_tags[k] = tags[i]
        else:
            s.sphere_data["radius"][k] = col["radius"]; s.sphere_tags[k] = tags[i]
    assert s.fits_reference() and tags.max() < 65536
    return EdgeScene(name, s, clusters, col_cluster)


TAILS = (1, 2, 7, 8, 9, 31, 33, 257, 1025, 4000)


def tail_scene(n):
    kinds = tail_kinds()
    clusters = [case("tail", i, kinds[i % len(kinds)], True if i % len(kinds) != 2 else False) for i in range(n)]
    return assemble("tail_%d" % n, clusters, seed=1000 + n)


def edge_scenes():
    """The edge-case scenes: everything that can share a scene in one, then one scene per case that needs the origin."""
    allc = box_box_cases() + main_cpp_cases() + box_sphere_cases() + sphere_sphere_cases() + tag_body_cases()
    ordinary = [c for c in allc if not c["origin"]]
    out = [assemble("edges", ordinary, seed=1)]
    for k, c in enumerate(c for c in allc if c["origin"]):
        out.append(assemble("origin_%d" % k, [c], seed=2 + k))
    return out


def all_scenes():
    return edge_scenes() + [tail_scene(n) for n in TAILS]


# ---------------- comparing a collide() output with the recorded one ----------------
def golden_of(g, es):
    """The recorded collide() output of scene `es` in the reference's layout."""
    p = es.name + "/"
    return dict(count=int(g[p + "count"][0]), data=g[p + "data"], a=g[p + "bodies_a"], b=g[p + "bodies_b"], tags=g[p + "tags"],
                sleeping=g[p + "sleeping"], active=g[p + "active"], inputs=g[p + "inputs"], digests=g[p + "digests"])


def collide_differences(es, want, view):
    """`view`: contacts_view() of a widened implementation.  Returns a list of messages (empty if bit-identical), each naming the family
    and case of the first differing contact."""
    from nudge_b200 import abi
    errs = []
    if not np.array_equal(want["inputs"], es.input_digest()):
        return ["%s: the generated scene differs from the one recorded (tests/np_edge_cases.py changed without re-recording)" % es.name]
    if view["count"] != want["count"]:
        cl = es.cluster_of_tag()
        got_cl = np.bincount(cl[(np.asarray(view["tags"], np.uint64) & np.uint64(0xffff)).astype(np.int64)], minlength=len(es.clusters))
        want_cl = np.bincount(cl[((want["tags"] >> np.uint64(32)) & np.uint64(0xffff)).astype(np.int64)], minlength=len(es.clusters))
        bad = np.nonzero(got_cl != want_cl)[0]
        return ["%s: %d contacts, the reference made %d; first differing cluster: %s (%d vs %d contacts)" %
                (es.name, view["count"], want["count"], es.describe(bad[0]), got_cl[bad[0]], want_cl[bad[0]])]
    tags = abi.wide_tag_to_ref(view["tags"], view["features"])
    cl = es.cluster_of_tag()[((want["tags"] >> np.uint64(32)) & np.uint64(0xffff)).astype(np.int64)]
    fields = [("data", view["data"].view(np.uint32).reshape(len(tags), 8), want["data"].view(np.uint32).reshape(len(tags), 8)),
              ("bodies.a", view["bodies"]["a"], want["a"]), ("bodies.b", view["bodies"]["b"], want["b"]), ("tags", tags, want["tags"])]
    for name, got, ref in fields:
        diff = got != ref
        if diff.ndim > 1:
            diff = diff.any(axis=1)
        bad = np.nonzero(diff)[0]
        if len(bad):
            i = bad[0]
            g_, r_ = got[i], ref[i]
            if name == "data":
                g_, r_ = got[i].view(np.float32), ref[i].view(np.float32)
            errs.append("%s: %s differs in %d of %d contacts; first: contact %d of %s\n   want %s\n   got  %s" %
                        (es.name, name, len(bad), len(tags), i, es.describe(cl[i]), r_, g_))
    if not np.array_equal(abi.wide_pair_to_ref(view["sleeping"]), want["sleeping"]):
        errs.append("%s: sleeping pairs differ" % es.name)
    if not np.array_equal(np.asarray(view["active"], np.uint32), want["active"]):
        errs.append("%s: active bodies differ" % es.name)
    return errs
