"""Joint rows against what they mean (tests/joint_geometry.py, float64 geometry independent of the restatements): every row of the numpy
restatement (tests/joint_dof_ref.py, which the device matches byte for byte) has the Jacobian of the coordinate it constrains, the bias its
coordinate's true value asks for, and the drive the position the download reports, over seeded random poses of every type and flag
combination, over the whole legal range of the angle limits, and at listed edge poses.  tests/test_gpu_joint_geometry.py applies the same
checks to the device's rows.

Tolerances (float32 eps = 2^-23 = 1.19e-7):
- Jacobian, on the manifold: every row's J v is the exact derivative of its coordinate there, so what is left is the float32 rounding of
  the row's components (each a product or cross product of float32 values, a few eps relative to |J|) and the O(h^2) central difference
  (h = 1e-4: about 1e-8 |v| per unit of lever arm).  Bound: 1e-5 * sum_k |J_k| |v_k| over the row's four parts (lever arms included),
  a distance row's direction err / dist turns by err's rounding over dist (4 eps (|pa| + |ra| + |pb| + |rb|) / dist of the bound's |J| |v|),
  and for a slider's rows 4 eps (|err| + |pa| + |ra| + |pb| + |rb|) |omega| more: their lever sa = ra - err carries err's rounding.
- Jacobian, off the manifold by a rotation e (radians) between the bodies: the angular rows' Jacobians are those of the coordinate at the
  manifold, and the rate of the true coordinate differs from them through terms like (omega x e), of size |e| |omega| per body.  Bound:
  2 |e| (|omega_a| + |omega_b|) on top of the rounding bound; the point, slider and distance rows are exact derivatives at any pose.
- The twist row is the exception on the manifold: its Jacobian is the hinge Jacobian about u, which is the twist's derivative only while the
  swing is 0.  Turning a by omega about n x u (n the swing axis) moves the twist at tan(swing / 2) |omega|, and the same holds on b's side, so
  the twist rows are held to tan(swing / 2) (|omega_a| + |omega_b|) more (asserted tight below: the bound is reached).
- Bias of an equality row: k C with C from float32 positions: the anchor error wa - wb cancels float32 values of size |p| + |r|, so its
  error is a few eps times |pa| + |ra| + |pb| + |rb|: bound k (4 eps (|pa| + |ra| + |pb| + |rb|) + 1e-6 |C|).  At 1e4 from the origin that is
  about 1e-2 k, the cancellation the float32 positions carry, not a property of the rows.
- Angle limits: sh, ch carry a few eps and the limits' pairs one ulp, so C is within 2e-6 of its exact value; the true angle is measured at
  the same float32 poses.  Inside: (2/pi) min(d, pi) - 2e-6 <= C <= d + 2e-6; past the bound C < 0 with the same bounds on |C|.
- Positions: within 1e-5 rad of the float64 angles, outside a 1e-4 band around +-pi where the angle wraps.
- Near a swing of pi the twist is ill-conditioned: its pair is (sh, ch) / cs with cs = cos(swing / 2), so the twist's positions and limit
  measures get 4 eps / cs more, and the cone row's direction, g / |g| with |g| = sin(swing), 4 eps / sin(swing) of |J| |v|."""
import numpy as np
import pytest
from scipy.spatial.transform import Rotation

import nudge_b200
from tests import joint_dof_ref as dof
from tests import joint_geometry as geo

DT = np.float32(1.0 / 60.0)
EPS = float(np.finfo(np.float32).eps)
ANGLE_TOL = 2e-6
BALL, HINGE, FIXED, DISTANCE = geo.BALL, geo.HINGE, geo.FIXED, geo.DISTANCE
L, M, BR, S, CN, TW = geo.LIMIT, geo.MOTOR, geo.BREAKABLE, geo.SLIDE, geo.CONE, geo.TWIST
COMBOS = [(BALL, 0), (BALL, CN), (BALL, TW), (BALL, CN | TW), (HINGE, 0), (HINGE, L), (HINGE, M), (HINGE, L | M), (FIXED, 0),
          (FIXED, S), (FIXED, S | L), (FIXED, S | M), (FIXED, S | L | M), (DISTANCE, 0), (DISTANCE, L)]


def drive(joint, flags, **kw):
    d = np.zeros(1, nudge_b200.JOINT_DRIVE)[0]
    d["joint"], d["flags"], d["break_force"], d["break_torque"] = joint, flags, np.inf, np.inf
    for k, v in kw.items():
        d[k] = v
    return d


def random_drive(typ, flags, rng, coordinate):
    """A drive of `flags` (BREAKABLE added at random, with infinite thresholds) with random limits around the joint's coordinate."""
    kw = dict(motor_speed=rng.normal() * 2.0, max_motor_torque=rng.random() * 5.0)
    if flags & CN:
        kw = dict(cone=rng.uniform(0.05, np.pi))
    if flags & (L | TW):
        if typ in (HINGE, BALL):
            kw["lower"], kw["upper"] = np.sort(rng.uniform(-np.pi, np.pi, 2))
        else:
            kw["lower"], kw["upper"] = np.sort(coordinate + rng.normal(size=2))
            if typ == DISTANCE:
                kw["lower"], kw["upper"] = max(kw["lower"], 0.0), max(kw["upper"], 0.0)
    return drive(0, flags | (BR if rng.random() < 0.3 else 0), **kw)


def random_joint(typ, flags, rng, b=True, off=0.0, far=0.0):
    """A joint of `typ` with a drive of `flags` at a random legal pose (tests/joint_geometry.place)."""
    kw = dict(b=b, off=off, far=far)
    if typ in (HINGE, BALL):
        kw["coordinate"] = rng.uniform(-np.pi, np.pi)
    if typ == BALL:
        kw["swing"] = rng.uniform(0.0, 2.5) if rng.random() < 0.7 else 0.0
    if typ == FIXED and flags & S:
        kw["coordinate"] = rng.normal() * 2.0
    if typ == DISTANCE:
        kw["coordinate"] = rng.uniform(0.2, 3.0)
    j, xf = geo.place(typ, rng, **kw)
    return j, random_drive(typ, flags, rng, kw.get("coordinate", 0.0)) if flags else None, xf


def rows_of(j, d, xf, dt=DT):
    """The restated rows of joint j with drive d (None: no drive) in solve order, and its drive table entry (None without a drive)."""
    joints = np.array([j])
    if d is None:
        return dof.joint_rows(joints, xf, dt), None
    table, imp = dof.drive_table(joints, [d])
    rows = dof.joint_rows(joints, xf, dt, table, imp)
    return rows[dof.solve_order(joints, table)], table[0]


def targets(j, flags, d):
    """One entry per row of joint j in solve order: (coordinate of geo.coordinates' dict whose derivative J v is, whether it is an angle,
    kind, the true value the bias is a function of).  kind: "eq" (bias = k C), "lo", "hi" (limit rows on the distance to their stop),
    "motor", "none" (a row that applies nothing)."""
    typ = int(j["type"])
    out = []
    if typ == DISTANCE:
        out.append((lambda c: c["distance"], False, "none" if flags & L else "eq", lambda c: c["distance"] - float(np.float32(j["length"]))))
        if flags & L:
            out.append((lambda c: c["distance"], False, "lo", lambda c: c["distance"] - float(d["lower"])))
            out.append((lambda c: -c["distance"], False, "hi", lambda c: float(d["upper"]) - c["distance"]))
        return out
    if flags & S:
        for r in range(3):
            # the slider's point rows measure wa - wb across the basis that turns with a
            def along(c, r=r):
                return c["anchor_error"] @ c["Ra"].apply(c["t_a"][r])
            out.append((along, False, "none" if r == 2 else "eq", along))
    else:
        for e in range(3):
            out.append((lambda c, e=e: c["anchor_error"][e], False, "eq", lambda c, e=e: c["anchor_error"][e]))
    if typ == HINGE:
        for r in range(2):
            def mis(c, r=r):
                return -(c["misalignment"] @ c["t"][r])
            out.append((mis, False, "eq", mis))
    if typ == FIXED:
        for e in range(3):
            out.append((lambda c, e=e: c["fixed"][e], False, "eq", lambda c, e=e: c["fixed"][e]))
    key = "s" if flags & S else "twist" if typ == BALL else "theta"
    if flags & (M | CN):
        if flags & CN:
            out.append((lambda c: -c["swing"], True, "lo", lambda c: float(d["cone"]) - c["swing"]))
        else:
            out.append((lambda c: c[key], typ == HINGE, "motor", None))
    if flags & (L | TW):
        out.append((lambda c: c[key], key != "s", "lo", lambda c: c[key] - float(d["lower"])))
        out.append((lambda c: -c[key], key != "s", "hi", lambda c: float(d["upper"]) - c[key]))
    return out


def _norm(x):
    return float(np.linalg.norm(np.asarray(x, np.float64)))


def check_joint(j, d, xf, rows, entry, rng, off=0.0, dt=DT, pos_tol=4.0, where="", h=1e-4):
    """Asserts every row of joint j (solve order) against the float64 geometry at xf: Jacobian, bias and the reported position.  off: how
    far the pose was placed off the manifold (radians and length units).  pos_tol: the tolerance of equality biases, in units of eps times
    the positions' scale (see the module's docstring).  Returns the worst Jacobian error of the twist rows over its bound (for the test that
    the bound is tight)."""
    flags = int(d["flags"]) if d is not None else 0
    if entry is not None and entry["broken"]:
        return 0.0
    a, b = int(j["a"]), int(j["b"])
    poses = (*geo.pose(xf, a), *geo.pose(xf, b))
    c0 = geo.coordinates(j, *poses)
    typ = int(j["type"])
    tg = targets(j, flags, d)
    assert len(tg) == len(rows), where
    Ra = poses[1]
    # the row directions that a row holds fixed in the world (HINGE's t_i) or in a's frame (the slider's t1, t2, u)
    t_world = [np.asarray(rows["ang_a"][3 + r], np.float64) for r in range(2)] if typ == HINGE else None
    t_a = [Ra.inv().apply(np.asarray(rows["lin_a"][r], np.float64)) for r in range(3)] if flags & S else None

    def values(*P):
        c = geo.coordinates(j, *P)
        c["t"], c["t_a"] = t_world, t_a
        return np.array([fn(c) for fn, *_ in tg])
    zero = np.zeros(3)
    vel = (rng.normal(size=3), rng.normal(size=3), rng.normal(size=3) if b else zero, rng.normal(size=3) if b else zero)
    angle = np.array([t[1] for t in tg])
    rate = geo.derivative(values, poses, vel, h=h, angle=angle)
    c0["t"], c0["t_a"] = t_world, t_a
    k = float(np.float32(j["beta"]) / dt)
    scale = _norm(poses[0]) + _norm(c0["ra"]) + _norm(poses[2]) + _norm(c0["rb"])
    worst_twist = 0.0
    # the twist pair is (sh, ch) / cs with cs = cos(swing / 2): a few eps of absolute error in sh and ch become 4 eps / cs of twist
    atol = ANGLE_TOL + (4.0 * EPS / np.cos(0.5 * c0["swing"]) if typ == BALL and flags & TW else 0.0)
    for i, ((fn, is_angle, kind, truth), r) in enumerate(zip(tg, rows)):
        what = "%s row %d (%s)" % (where, i, kind)
        J = [np.asarray(r[x], np.float64) for x in ("lin_a", "ang_a", "lin_b", "ang_b")]
        jv = sum(x @ v for x, v in zip(J, vel))
        size = sum(_norm(x) * _norm(v) for x, v in zip(J, vel))
        omega = _norm(vel[1]) + _norm(vel[3])
        rotational = typ != DISTANCE and i >= 3 and not (flags & S and kind in ("lo", "hi", "motor"))
        tol = 1e-5 * size + 1e-9 + (2.0 * off * omega if rotational else 0.0)
        if typ == DISTANCE and c0["distance"] > 0:   # n = err / dist: err's rounding, 4 eps scale, turns n by that over dist
            tol += 4.0 * EPS * scale / c0["distance"] * size
        if flags & S and not rotational:   # the lever sa = ra - err: cross(sa, t) cancels float32 values of size |err|
            tol += 4.0 * EPS * (_norm(c0["anchor_error"]) + scale) * omega
        if typ == BALL and flags & CN and i == 3:
            if c0["swing"] < 1e-3:
                continue   # the cone row on an (almost) zero swing: the swing is not differentiable there; see the edge test
            # n = g / |g| with |g| = sin(swing) from float32 values of size 1: a few eps / sin(swing) of direction
            tol += 4.0 * EPS / np.sin(c0["swing"]) * size
        if typ == BALL and flags & TW and kind in ("lo", "hi") and not (flags & CN and i == 3):
            bound = tol + np.tan(0.5 * c0["swing"]) * omega
            worst_twist = max(worst_twist, abs(jv - rate[i]) / max(bound, 1e-12) if c0["swing"] > 0.1 else 0.0)
            tol = bound
        assert abs(jv - rate[i]) <= tol, (what, jv, rate[i], tol)
        bias = float(r["bias"])
        if kind == "eq":
            C = truth(c0)
            btol = k * (pos_tol * EPS * scale + 1e-6 * abs(C)) + 1e-9
            assert abs(bias - k * C) <= btol, (what, bias, k * C, btol)
        elif kind == "motor":
            lim = np.float32(d["max_motor_torque"]) * dt
            assert bias == -np.float32(d["motor_speed"]) and r["lo"] == -lim and r["hi"] == lim, what
        elif kind in ("lo", "hi"):
            dist = truth(c0)
            assert r["lo"] == 0 and r["hi"] == np.inf, what
            C = bias * float(dt) if bias > 0 else bias / k
            if is_angle:
                if key_near_pi(c0, typ, flags):
                    continue
                lower_bound = (2.0 / np.pi) * min(abs(dist), np.pi)
                if dist > atol:
                    assert 0 < C <= dist + atol and C >= lower_bound - atol, (what, C, dist)
                elif dist < -atol:
                    assert C < 0 and -C <= -dist + atol and -C >= lower_bound - atol, (what, C, dist)
                else:
                    assert abs(C) <= 2 * atol, (what, C, dist)
            else:
                ltol = 4 * EPS * (scale + abs(float(d["lower"])) + abs(float(d["upper"]))) + 1e-9
                assert abs(C - dist) <= ltol * (1.0 if bias <= 0 else 1.0 + 1e-6), (what, C, dist, ltol)
        else:
            assert r["lo"] == 0 and r["hi"] == 0, what
    if entry is not None and flags & (L | S | CN | TW):
        got = float(dof.drive_position(typ, flags, entry["position"]))
        want = c0["s"] if flags & S else c0["distance"] if typ == DISTANCE else c0["theta"] if typ == HINGE else \
            c0["twist"] if flags & TW else c0["swing"]
        if flags & S or typ == DISTANCE:
            assert abs(got - want) <= 4 * EPS * (scale + abs(want)), (where, got, want)
        elif abs(want) < np.pi - 1e-4:   # off the manifold the angles' definitions part by O(off^2)
            assert abs(got - want) <= 1e-5 + (atol - ANGLE_TOL) + off * off, (where, got, want)
    return worst_twist


def key_near_pi(c, typ, flags):
    """Whether the joint's angle lies in the band around +-pi where the angle wraps and the limit measure's two ends meet."""
    x = c["twist"] if typ == BALL and flags & TW else c["theta"] if typ == HINGE else 0.0
    return abs(x) > np.pi - 1e-5


def _check(j, d, xf, rng, **kw):
    rows, entry = rows_of(j, d, xf)
    return check_joint(j, d, xf, rows, entry, rng, **kw)


@pytest.mark.parametrize("typ,flags", COMBOS)
def test_rows_on_the_manifold(typ, flags):
    rng = np.random.default_rng(100 + 8 * typ + flags)
    for n in range(40):
        j, d, xf = random_joint(typ, flags, rng, b=n % 4 != 0)
        _check(j, d, xf, rng, where="%d/%d #%d" % (typ, flags, n))


@pytest.mark.parametrize("off", [1e-3, 1e-2, 0.1])
def test_rows_off_the_manifold(off):
    rng = np.random.default_rng(int(off * 1e4))
    for typ, flags in COMBOS:
        for n in range(8):
            j, d, xf = random_joint(typ, flags, rng, b=n % 4 != 0, off=off)
            _check(j, d, xf, rng, off=off, where="%d/%d #%d off %g" % (typ, flags, n, off))


def test_twist_rows_reach_their_stated_bound():
    """The twist rows' Jacobian misses the twist's rate by up to tan(swing / 2) |omega| (module docstring): the bound is reached, not loose."""
    rng = np.random.default_rng(7)
    worst = max(_check(*random_joint(BALL, TW, rng), rng) for _ in range(60))
    assert 0.3 < worst <= 1.0, worst


def _limit_c(rows, k):
    """C of the lower and upper angle limit rows (the last two), recovered from their biases."""
    return [float(b) * float(DT) if b > 0 else float(b) / k for b in rows["bias"][-2:]]


@pytest.mark.parametrize("typ", [HINGE, BALL])
def test_wide_range_limits_over_the_whole_legal_range(typ):
    """theta - lower and upper - theta over [-2 pi, 2 pi]: lower and upper anywhere in [-pi, pi], theta (or the twist, under a swing of 0.7)
    anywhere in (-pi, pi).  Inside the range 0 < C <= d and C >= (2/pi) min(d, pi); past the bound C < 0 with the same bounds on |C|; C
    increasing in d.  The sine alone, 2 sin(d / 2), breaks the lower bound and the monotony wherever d > pi."""
    rng = np.random.default_rng(11 + typ)
    pi32 = float(np.float32(np.pi))
    stops = np.concatenate([np.linspace(-np.pi, np.pi, 13)[1:-1], [-pi32, pi32, -3.1, 3.1]])
    angles = np.concatenate([np.linspace(-np.pi + 1e-3, np.pi - 1e-3, 61), [0.0, np.pi / 2, -np.pi / 2, 3.1, -3.1]])
    flags = L if typ == HINGE else TW
    for stop in stops:
        seen = {0: [], 1: []}
        for x in angles:
            j, xf = geo.place(typ, rng, b=bool(rng.random() < 0.5), coordinate=x, swing=0.7 if typ == BALL else 0.0)
            for side, (lo, hi) in enumerate(((stop, pi32), (-pi32, stop))):
                d = drive(0, flags, lower=lo, upper=hi)
                rows, entry = rows_of(j, d, xf)
                _check(j, d, xf, rng, where="stop %g angle %g side %d" % (stop, x, side))
                c = geo.coordinates(j, *geo.pose(xf, 1), *geo.pose(xf, int(j["b"])))
                a = c["theta"] if typ == HINGE else c["twist"]
                dist = a - float(np.float32(lo)) if side == 0 else float(np.float32(hi)) - a
                seen[side].append((dist, _limit_c(rows, float(np.float32(0.2) / DT))[side]))
        for side in (0, 1):
            got = np.array(sorted(seen[side]))
            assert (np.diff(got[:, 1]) >= -ANGLE_TOL).all(), (stop, side)
            wide = got[:, 0] > np.pi
            assert (got[wide, 1] >= 2.0 - ANGLE_TOL).all(), (stop, side, got[wide][:3])


def _ux(x):
    """A unit axis with x component x and equal y and z."""
    r = np.sqrt((1.0 - x * x) / 2.0)
    return np.array([x, r, r])


def test_edge_poses():
    rng = np.random.default_rng(21)
    pi32 = float(np.float32(np.pi))
    # within 1e-3 of +-pi d.w changes sign and flips the pair; closer still, the float32 poses' 1e-7 off the hinge manifold make the true
    # angle's rate ill-conditioned (it moves by about e |omega| / (pi - |theta|) for an offset e), which is a property of the angle
    near = [0.0, np.pi / 2, -np.pi / 2, np.pi - 1e-3, -np.pi + 1e-3]
    ranges = [(-pi32, pi32), (0.3, 0.3), (-1.5, 1.64), (-1.6, 1.6), (-pi32, -pi32), (pi32, pi32), (-3.1, 3.1)]
    for typ, flags in ((HINGE, L | M), (BALL, TW), (BALL, CN | TW)):
        for x in near:
            for lo, hi in ranges:
                for b in (True, False):
                    j, xf = geo.place(typ, rng, b=b, coordinate=x, swing=0.4 if typ == BALL else 0.0)
                    d = drive(0, flags, lower=lo, upper=hi, cone=1.0) if flags & CN else drive(0, flags, lower=lo, upper=hi, motor_speed=1.0, max_motor_torque=2.0)
                    _check(j, d, xf, rng, where="%d/%d at %g in [%g, %g]" % (typ, flags, x, lo, hi))
    # the hinge basis switch at |u.x| = 0.57735, and the slider's, on both sides
    for ux in (0.57735 - 1e-6, 0.57735 + 1e-6, -0.57735 - 1e-6, -0.57735 + 1e-6):
        for typ, flags, x in ((HINGE, L | M, 1.0), (FIXED, S | L | M, 0.5)):
            j, xf = geo.place(typ, rng, coordinate=x, u=_ux(ux))
            _check(j, drive(0, flags, lower=-2.0, upper=2.0, motor_speed=1.0, max_motor_torque=1.0), xf, rng, where="basis %g" % ux)
    # swing 0: the cone row is a zero row or a unit one with C = cone; swing within 1e-3 of pi: cs -> 0
    for swing in (0.0, 1e-6, np.pi - 1e-3, np.pi - 1e-4):
        for tw in (0.0, 1.0, -2.5):
            j, xf = geo.place(BALL, rng, coordinate=tw, swing=swing)
            d = drive(0, CN | TW, cone=0.5, lower=-3.0, upper=3.0)
            rows, _ = rows_of(j, d, xf)
            n = np.asarray(rows["ang_b"][3], np.float64)
            assert np.array_equal(n, -np.asarray(rows["ang_a"][3], np.float64)) and (not n.any() or abs(np.linalg.norm(n) - 1.0) < 1e-6)
            if swing < 1e-3:
                assert abs(float(rows["bias"][3]) * float(DT) - 2 * np.sin(0.25)) < 1e-5   # C = 2 sin((cone - 0) / 2)
            else:
                _check(j, d, xf, rng, where="swing %g twist %g" % (swing, tw), h=1e-6)   # h well inside the 1e-3 to the pole
    # a distance joint with coincident anchors: the row on (0, 1, 0), bias k (0 - length)
    for length, flags in ((0.0, 0), (0.5, 0), (0.0, L)):
        j, xf = geo.place(DISTANCE, rng, b=False, coordinate=0.0)
        j["length"], j["anchor_a"], j["anchor_b"] = length, 0.0, xf["position"][1]   # wa = wb exactly in float32
        d = drive(0, L, lower=0.0, upper=1.0) if flags else None
        rows, _ = rows_of(j, d, xf)
        assert tuple(rows["lin_a"][0]) == (0.0, 1.0, 0.0) and tuple(rows["lin_b"][0]) == (0.0, -1.0, 0.0)
        k = np.float32(0.2) / DT
        assert rows["bias"][0] == k * np.float32(-length)
        if flags:
            assert rows["bias"][1] == 0.0 and rows["bias"][2] == np.float32(1.0) / DT
    # sliders far along their axis, and every type 1e4 from the origin, where float32 positions carry 1e-3 of cancellation in wa - wb
    for s in (-1e3, -10.0, 10.0, 1e3):
        j, xf = geo.place(FIXED, rng, coordinate=s)
        _check(j, drive(0, S | L | M, lower=-2e3, upper=2e3, motor_speed=1.0, max_motor_torque=1.0), xf, rng, where="s %g" % s)
    for typ, flags in COMBOS:
        for n in range(4):
            j, d, xf = random_joint(typ, flags, rng, b=n % 2 == 0, far=1e4)
            _check(j, d, xf, rng, where="%d/%d far #%d" % (typ, flags, n))
