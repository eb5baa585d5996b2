"""What a joint's rows mean, in float64 from the bodies' poses (include/nudge_b200.h, Joints and Joint drives) — TEST INFRASTRUCTURE ONLY.

An account of each joint's coordinates independent of the restatements (oracle/joints_ref.py, tests/joint_drives_ref.py,
tests/joint_dof_ref.py) and of their half-angle arithmetic: rotations are scipy.spatial.transform.Rotation, vectors float64.  A pose is
(p, R) per body; the static world (b = 0) is the origin with the identity, so b's anchor is a world point and axis_b a world axis.

Coordinates of one joint (`coordinates`):
  anchor_error   wa - wb (BALL, HINGE and FIXED point rows)
  misalignment   cross(u, w), u = R_a axis_a and w = R_b axis_b (HINGE's angular rows)
  rotvec         the rotation vector of D = R_a R_rel R_b^T, and fixed = 2 * the vector part of D's quaternion with w >= 0 (FIXED)
  theta          b's rotation relative to a about u: D turns b back onto a, so theta = -(rotvec . u); b turning positively about u
                 relative to a increases it
  swing          arccos(u . D u) (as atan2(|u x D u|, u . D u));  twist: the angle about u of swing^-1 D, negated like theta (the
                 swing is the shortest rotation that takes u to D u)
  s, offset      (wb - wa) . u and the part of wb - wa perpendicular to u (FIXED + SLIDE)
  distance       |wa - wb|
`derivative` differentiates any function of the poses along body velocities (v, omega) by float64 central differences, rotations advancing
as exp(omega h) R.  `place` builds a joint and its two poses exactly on the manifold of the joint's equalities in float64 (or a chosen
distance off it), then rounds everything to float32 as the device holds it."""
import numpy as np
from scipy.spatial.transform import Rotation

import nudge_b200
from nudge_b200 import scenes

BALL, HINGE, FIXED, DISTANCE = 0, 1, 2, 3
LIMIT, MOTOR, BREAKABLE, SLIDE, CONE, TWIST = 1, 2, 4, 16, 32, 64
IDENTITY = Rotation.identity()


def pose(xf, i):
    """Body i's pose (p, R) in float64 from a TRANSFORM array; body 0 is the world."""
    if i == 0:
        return np.zeros(3), IDENTITY
    return xf["position"][i].astype(np.float64), Rotation.from_quat(xf["rotation"][i].astype(np.float64))


def wrap(x):
    """x wrapped into [-pi, pi)."""
    return (np.asarray(x, np.float64) + np.pi) % (2.0 * np.pi) - np.pi


def coordinates(j, pa, Ra, pb, Rb):
    """The coordinates of joint j (nudge_b200.JOINT) at the poses (pa, Ra) of a and (pb, Rb) of b (the world: zeros, IDENTITY)."""
    f64 = lambda k: np.asarray(j[k], np.float64)
    ra, rb = Ra.apply(f64("anchor_a")), Rb.apply(f64("anchor_b"))
    wa, wb = pa + ra, pb + rb
    u, w = Ra.apply(f64("axis_a")), Rb.apply(f64("axis_b"))
    u, w = u / np.linalg.norm(u), w / np.linalg.norm(w)   # the float32 axes are unit within a few eps
    D = Ra * Rotation.from_quat(f64("rel_rotation")) * Rb.inv()
    q = D.as_quat()
    q = -q if q[3] < 0 else q
    rv = D.as_rotvec()
    Du = D.apply(u)
    axis = np.cross(u, Du)
    n = np.linalg.norm(axis)
    swing = np.arctan2(n, u @ Du)
    S = Rotation.from_rotvec(axis / n * swing) if n > 0 else IDENTITY
    twist = -((S.inv() * D).as_rotvec() @ u)
    rel = wb - wa
    s = rel @ u
    return dict(Ra=Ra, ra=ra, rb=rb, wa=wa, wb=wb, u=u, anchor_error=wa - wb, misalignment=np.cross(u, w), rotvec=rv, fixed=2.0 * q[:3],
                theta=-(rv @ u), swing=swing, twist=twist, s=s, offset=rel - s * u, distance=np.linalg.norm(wa - wb))


def advance(p, R, v, omega, h):
    """A pose moved for time h at linear velocity v and angular velocity omega (world frame)."""
    return p + np.asarray(v, np.float64) * h, Rotation.from_rotvec(np.asarray(omega, np.float64) * h) * R


def derivative(fn, poses, vel, h=1e-4, angle=False):
    """d/dt of fn(pa, Ra, pb, Rb) at `poses` = (pa, Ra, pb, Rb) along vel = (va, wa, vb, wb), by float64 central differences (O(h^2));
    `angle` (a bool or a mask over fn's values): those differences are wrapped into [-pi, pi)."""
    pa, Ra, pb, Rb = poses
    va, wa, vb, wb = vel
    plus = fn(*advance(pa, Ra, va, wa, h), *advance(pb, Rb, vb, wb, h))
    minus = fn(*advance(pa, Ra, va, wa, -h), *advance(pb, Rb, vb, wb, -h))
    d = np.asarray(plus, np.float64) - np.asarray(minus, np.float64)
    return np.where(angle, wrap(d), d) / (2.0 * h)


def _unit(rng):
    v = rng.normal(size=3)
    return v / np.linalg.norm(v)


def _perpendicular(u, rng):
    v = np.cross(u, _unit(rng))
    return v / np.linalg.norm(v)


def place(typ, rng, b=True, coordinate=None, swing=0.0, swing_axis=None, u=None, off=0.0, far=0.0, anchors=1.0):
    """A joint of type `typ` between body a (1) and body b (2, or the world when not b), and its float32 transforms (3 bodies, the world
    first), with the joint's equalities exact in float64 before the rounding:
      HINGE     axes aligned, anchors coincident, theta = coordinate
      BALL      anchors coincident, swing `swing` about swing_axis (perpendicular to u; random if None), twist = coordinate
      FIXED     the rest rotation exact; with coordinate not None a slider: anchors on the line along u, s = coordinate
      DISTANCE  |wa - wb| = coordinate = the joint's length
    u: the world axis (axis_a; random if None).  off: b moved by `off` along a random direction and turned by `off` rad about another (the
    joint that far off its manifold).  far: the bodies placed about `far` from the origin.  anchors: the anchors' scale."""
    j = np.zeros(1, nudge_b200.JOINT)[0]
    j["type"], j["a"], j["b"], j["beta"] = typ, 1, 2 if b else 0, 0.2
    u = _unit(rng) if u is None else np.asarray(u, np.float64) / np.linalg.norm(u)
    rel = Rotation.random(random_state=rng)
    x = 0.0 if coordinate is None else float(coordinate)
    if typ == HINGE:
        D = Rotation.from_rotvec(-x * u)
    elif typ == BALL:
        n = _perpendicular(u, rng) if swing_axis is None else np.asarray(swing_axis, np.float64)
        D = Rotation.from_rotvec(swing * n) * Rotation.from_rotvec(-x * u)
    else:
        D = IDENTITY
    Rb = Rotation.random(random_state=rng) if b else IDENTITY
    Ra = D * Rb * rel.inv()   # D = Ra rel Rb^T
    centre = far * _unit(rng) if far else rng.normal(size=3) * 2.0
    pa = centre + rng.normal(size=3)
    anchor_a = rng.normal(size=3) * anchors
    wa = pa + Ra.apply(anchor_a)
    if typ == DISTANCE:
        wb = wa + _unit(rng) * x
    elif typ == FIXED and coordinate is not None:
        wb = wa + x * u
    else:
        wb = wa.copy()
    anchor_b = rng.normal(size=3) * anchors if b else wb
    pb = wb - Rb.apply(anchor_b) if b else np.zeros(3)
    j["anchor_a"], j["anchor_b"] = anchor_a, anchor_b
    j["axis_a"], j["axis_b"] = Ra.inv().apply(u), Rb.inv().apply(u)
    j["rel_rotation"] = rel.as_quat()
    j["length"] = x if typ == DISTANCE else 0.0
    if off:
        # b (a when b is the world) turned about its anchor and moved: the anchors' and the axes' errors both of order `off`
        turn, move = Rotation.from_rotvec(off * _unit(rng)), off * _unit(rng)
        if b:
            Rb = turn * Rb; pb = wb + move - Rb.apply(anchor_b)
        else:
            Ra = turn * Ra; pa = wa + move - Ra.apply(anchor_a)
    xf = np.zeros(3, scenes.TRANSFORM)
    xf["rotation"][:, 3] = 1.0
    xf["position"][1], xf["rotation"][1] = pa, Ra.as_quat()
    if b:
        xf["position"][2], xf["rotation"][2] = pb, Rb.as_quat()
    return j, xf
