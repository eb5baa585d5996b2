"""Spring rows against what they mean (tests/joint_geometry.py, float64 geometry independent of the restatements): every spring row of the
numpy restatement (tests/joint_spring_ref.py, which the device matches byte for byte) has the Jacobian of its coordinate, the C its
coordinate's true value gives, the softness and bounds of the soft step, and the spring the position the download reports; over seeded
random poses of every type (b on and off, anchors off the axis, off the manifold, far from the origin), hinge angles and targets at and
across the +-pi seam, and ball targets far from the joint's rotation.  tests/test_gpu_joint_springs.py applies check_spring to the device's
rows.

Tolerances, as tests/test_joint_geometry_ref.py derives them for the joints' own and drive rows:
- Jacobian: 1e-5 * sum_k |J_k| |v_k| + 1e-9; a HINGE row off the manifold by a rotation e also 2 |e| (|omega_a| + |omega_b|); a FIXED row
  (J_s, lever sa = ra - err) 4 eps (|err| + |pa| + |ra| + |pb| + |rb|) |omega| more; a DISTANCE row 4 eps scale / dist of |J| |v| more.
- BALL: the rows are FIXED's angular rows on the target rotation: J v = e . (omega_a - omega_b), while 2 d.e of d = R_a T R_b^T moves at
  d.w Omega + Omega x d.xyz with Omega = omega_a - d omega_b.  The two agree at the target and part by at most 2 phi (|omega_a| + |omega_b|)
  at an angle phi from it, which is the bound (the row is exact where the spring rests).
- C, recovered from the bias as (bias * den + damping * target_velocity) / stiffness: a linear coordinate within 4 eps of the positions'
  scale and its target; an angle's measure within 2e-6 (its pair and the target's pair carry a few eps); plus the recovery's own rounding,
  4 eps (|bias| den + damping |target_velocity|) / stiffness.
- Positions: within 4 eps of the scale for s and dist; within 1e-5 rad for the hinge angle (outside 1e-4 of +-pi, where it wraps) and the
  ball's angle from its target."""
import numpy as np
from scipy.spatial.transform import Rotation

import nudge_b200
from tests import joint_geometry as geo
from tests import joint_spring_ref as spr
from tests.test_joint_springs_ref import spring

DT = np.float32(1.0 / 60.0)
EPS = float(np.finfo(np.float32).eps)
ANGLE_TOL = 2e-6
BALL, HINGE, FIXED, DISTANCE = geo.BALL, geo.HINGE, geo.FIXED, geo.DISTANCE
PI32 = float(np.float32(np.pi))


def measure(d):
    """The angle measure of a difference d in [-2 pi, 2 pi] in float64: 2 sin(d / 2) while cos(d / 2) >= 0, then +-(4 - 2 |sin(d / 2)|)."""
    x = 0.5 * d
    s, c = np.sin(x), np.cos(x)
    return 2.0 * s if c >= 0 else np.sign(x) * (4.0 - 2.0 * abs(s))


def _norm(x):
    return float(np.linalg.norm(np.asarray(x, np.float64)))


def random_case(typ, rng, b=True, off=0.0, far=0.0, coordinate=None, target=None, near=False):
    """A joint of `typ` at a legal pose (geo.place) and a spring on it: random gains, target and target velocity (0 for a BALL).  A BALL
    target is a random rotation, or with `near` one within 0.3 rad of the joint's relative rotation."""
    kw = dict(b=b, off=off, far=far)
    if typ in (HINGE, BALL):
        kw["coordinate"] = rng.uniform(-np.pi, np.pi) if coordinate is None else coordinate
    if typ == BALL:
        kw["swing"] = rng.uniform(0.0, 2.5)
    if typ == FIXED:
        kw["coordinate"] = rng.normal() * 2.0 if coordinate is None else coordinate
    if typ == DISTANCE:
        kw["coordinate"] = rng.uniform(0.2, 3.0) if coordinate is None else coordinate
    j, xf = geo.place(typ, rng, **kw)
    x = kw.get("coordinate", 0.0)
    if typ == BALL:
        pa, Ra, pb, Rb = (*geo.pose(xf, 1), *geo.pose(xf, int(j["b"])))
        rel = Ra.inv() * Rb   # conj(q_a) q_b: the target at which the spring rests here
        t = (rel * Rotation.from_rotvec(rng.normal(size=3) * 0.1)) if near else Rotation.random(random_state=rng)
        t = t.as_quat()
    elif target is not None:
        t = target
    else:
        t = rng.uniform(-np.pi, np.pi) if typ == HINGE else x + rng.normal() if typ == FIXED else rng.uniform(0.0, 3.0)
    sp = spring(0, t, rng.uniform(1.0, 100.0), rng.uniform(0.0, 5.0), 0.0 if typ == BALL else rng.normal(),
                np.inf if rng.random() < 0.5 else rng.uniform(0.1, 20.0))
    return j, sp, xf


def rows_of(j, sp, xf, dt=DT):
    """The restated spring rows of joint j with spring sp, and its table entry (position written)."""
    joints = np.array([j])
    table, imp = spr.spring_table(joints, [sp])
    _, srows = spr.joint_rows(joints, xf, dt, None, None, table, imp)
    return srows, table[0]


def check_spring(j, sp, xf, srows, entry, rng, off=0.0, dt=DT, where="", h=1e-4):
    """Asserts every spring row of joint j against the float64 geometry at xf: Jacobian, C, softness, bounds, and the reported position."""
    typ, a, b = int(j["type"]), int(j["a"]), int(j["b"])
    poses = (*geo.pose(xf, a), *geo.pose(xf, b))
    c0 = geo.coordinates(j, *poses)
    assert len(srows) == spr.spring_row_count(typ), where
    tgt = np.asarray(sp["target"], np.float64)
    T = Rotation.from_quat(tgt) if typ == BALL else None

    def values(pa, Ra, pb, Rb):
        if typ == BALL:
            q = (Ra * T * Rb.inv()).as_quat()
            q = -q if q[3] < 0 else q
            return 2.0 * q[:3]
        c = geo.coordinates(j, pa, Ra, pb, Rb)
        return np.array([c["theta"] if typ == HINGE else c["s"] if typ == FIXED else c["distance"]])
    zero = np.zeros(3)
    vel = (rng.normal(size=3), rng.normal(size=3), rng.normal(size=3) if b else zero, rng.normal(size=3) if b else zero)
    rate = geo.derivative(values, poses, vel, h=h, angle=typ == HINGE)
    now = values(*poses)
    k, c, vt = (float(np.float32(sp[x])) for x in ("stiffness", "damping", "target_velocity"))
    den = float(np.float32(np.float32(c) + np.float32(dt * np.float32(k))))
    scale = _norm(poses[0]) + _norm(c0["ra"]) + _norm(poses[2]) + _norm(c0["rb"])
    omega = _norm(vel[1]) + _norm(vel[3])
    phi = (T.inv() * Rotation.from_matrix(poses[1].as_matrix()).inv() * poses[3]).magnitude() if typ == BALL else 0.0   # angle from the target
    for i, r in enumerate(srows):
        what = "%s spring row %d" % (where, i)
        J = [np.asarray(r[x], np.float64) for x in ("lin_a", "ang_a", "lin_b", "ang_b")]
        jv = sum(x @ v for x, v in zip(J, vel))
        size = sum(_norm(x) * _norm(v) for x, v in zip(J, vel))
        tol = 1e-5 * size + 1e-9
        if typ == HINGE:
            tol += 2.0 * off * omega
        if typ == FIXED:
            tol += 4.0 * EPS * (_norm(c0["anchor_error"]) + scale) * omega
        if typ == DISTANCE and c0["distance"] > 0:
            tol += 4.0 * EPS * scale / c0["distance"] * size
        if typ == BALL:
            tol += 2.0 * phi * omega
        assert abs(jv - rate[i]) <= tol, (what, jv, rate[i], tol)
        # the soft step's softness and bounds
        assert abs(float(r["softness"]) - 1.0 / (float(dt) * (c + float(dt) * k))) <= 1e-6 * float(r["softness"]), what
        lim = np.float32(np.float32(sp["max_force"]) * dt)
        assert r["lo"] == -lim and r["hi"] == lim, what
        # C from the bias against the coordinate's true value
        bias = float(r["bias"])
        C = (bias * den + c * vt) / k
        ctol = 4.0 * EPS * (abs(bias) * den + c * abs(vt)) / k
        if typ == HINGE:
            if abs(c0["theta"]) > np.pi - 1e-5:
                continue   # the angle wraps here, and the measure's two ends meet
            want = measure(c0["theta"] - float(np.float32(tgt[0])))
            ctol += ANGLE_TOL + off * off
            dd = abs(c0["theta"] - float(np.float32(tgt[0])))
            # never the short way round: |C| >= (2/pi) min(|d|, pi), with d the difference within [-2 pi, 2 pi], not wrapped
            assert abs(C) >= (2.0 / np.pi) * min(dd, np.pi) - ctol and np.sign(C) * np.sign(c0["theta"] - tgt[0]) >= 0 or abs(C) <= ctol, what
        elif typ == BALL:
            want = now[i]
            ctol += 8.0 * EPS
        else:
            want = now[0] - float(np.float32(tgt[0]))
            ctol += 4.0 * EPS * (scale + abs(float(tgt[0])) + abs(now[0]))
        assert abs(C - want) <= ctol, (what, C, want, ctol)
    got = float(spr.spring_position(typ, entry["position"]))
    if typ == HINGE:
        if abs(c0["theta"]) < np.pi - 1e-4:
            assert abs(got - c0["theta"]) <= 1e-5 + off * off, (where, got, c0["theta"])
    elif typ == BALL:
        assert abs(got - phi) <= 1e-5, (where, got, phi)
    else:
        want = c0["s"] if typ == FIXED else c0["distance"]
        assert abs(got - want) <= 4 * EPS * (scale + abs(want)), (where, got, want)


def cases(seed=41, n=40):
    """(joint, spring, transforms, off) over every type: random poses on and off the manifold and far from the origin, hinge angles and
    targets at and across the +-pi seam, ball targets far from and near the joint's rotation."""
    rng = np.random.default_rng(seed)
    out = []
    for typ in (BALL, HINGE, FIXED, DISTANCE):
        for m in range(n):
            off = (0.0, 0.0, 1e-3)[m % 3] if typ != BALL else 0.0
            far = 1e4 if m % 13 == 0 else 0.0
            j, sp, xf = random_case(typ, rng, b=m % 3 != 0, off=off if not far else 0.0, far=far, near=typ == BALL and m % 2 == 0)
            out.append((j, sp, xf, off if not far else 0.0))
    for x in (np.pi - 1e-3, -np.pi + 1e-3, np.pi - 0.1, -np.pi + 0.1, 2.0, -2.0, 0.0):
        for t in (PI32, -PI32, 3.0, -3.0, 1.5, -1.5, 0.0):
            j, sp, xf = random_case(HINGE, rng, b=bool(rng.random() < 0.5), coordinate=x, target=t)
            out.append((j, sp, xf, 0.0))
    return out


def test_spring_rows_against_the_float64_geometry():
    rng = np.random.default_rng(5)
    for n, (j, sp, xf, off) in enumerate(cases()):
        srows, entry = rows_of(j, sp, xf)
        check_spring(j, sp, xf, srows, entry, rng, off=off, where="case %d type %d" % (n, int(j["type"])))
