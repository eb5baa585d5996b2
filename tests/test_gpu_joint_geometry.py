"""The device's joint rows against what they mean (tests/joint_geometry.py, float64 geometry independent of the restatements): every row of
a few thousand joints of every type and flag combination, at random, edge, far and off-manifold poses, checked for its Jacobian, bias and
reported position by tests/test_joint_geometry_ref.check_joint; and behaviour measured in float64 from downloaded transforms: wide hinge
and twist ranges that do not brake at their far stop, pendulums against every kind of limit over graph replays, motors reaching their
speed with the header's sign, and blocked motors at their impulse bound."""
import numpy as np
import pytest
from scipy.spatial.transform import Rotation

import nudge_b200
from nudge_b200 import scenes
from oracle import joints_ref
from tests import joint_dof_ref as dof
from tests import joint_geometry as geo
from tests.gpu_util import side_stream, joint_rows
from tests.test_joint_geometry_ref import COMBOS, BALL, HINGE, FIXED, DISTANCE, L, M, S, CN, TW, drive, random_joint, check_joint

pytestmark = pytest.mark.gpu


def _scene(n, size=0.3, gravity=0.0):
    """n cubes of side 2 * size far above the ground (body 0), at rest, no damping."""
    s = scenes.demo_scene(n, 0, iterations=8, spread=200.0, height=10.0, seed=3)
    s.box_data["size"][1:] = size
    s.properties[1:] = scenes._box_props(s.box_data["size"][1:])
    s.transforms["rotation"][:] = (0.0, 0.0, 0.0, 1.0)
    s.momentum["velocity"][:] = 0.0; s.momentum["angular_velocity"][:] = 0.0
    s.gravity = np.float32(gravity); s.damping = np.float32(0.0)
    return s


def _poses():
    """(joint, drive or None, float32 transforms of the world, a and b) over every type and flag combination: random poses on the
    manifold, off it, far from the origin, and the edge poses of tests/test_joint_geometry_ref."""
    rng = np.random.default_rng(31)
    out = []
    for typ, flags in COMBOS:
        for n in range(120):
            off = (0.0, 0.0, 0.0, 1e-3, 1e-2)[n % 5]
            far = 1e4 if n % 11 == 0 else 0.0
            j, d, xf = random_joint(typ, flags, rng, b=n % 3 != 0, off=off if not far else 0.0, far=far)
            out.append((j, d, xf, off if not far else 0.0))
    pi32 = float(np.float32(np.pi))
    for typ, flags in ((HINGE, L | M), (BALL, TW), (BALL, CN | TW)):
        for x in (0.0, np.pi / 2, -np.pi / 2, np.pi - 1e-3, -np.pi + 1e-3):
            for lo, hi in ((-pi32, pi32), (0.3, 0.3), (-1.5, 1.64), (-1.6, 1.6), (-3.1, 3.1), (pi32, pi32)):
                j, xf = geo.place(typ, rng, b=bool(rng.random() < 0.5), coordinate=x, swing=0.4 if typ == BALL else 0.0)
                d = drive(0, flags, lower=lo, upper=hi, cone=1.0) if flags & CN else drive(0, flags, lower=lo, upper=hi, motor_speed=1.0, max_motor_torque=2.0)
                out.append((j, d, xf, 0.0))
    for ux in (0.57735 - 1e-6, 0.57735 + 1e-6):
        r = np.sqrt((1.0 - ux * ux) / 2.0)
        for typ, flags, x in ((HINGE, L | M, 1.0), (FIXED, S | L | M, 0.5)):
            j, xf = geo.place(typ, rng, coordinate=x, u=(ux, r, r))
            out.append((j, drive(0, flags, lower=-2.0, upper=2.0, motor_speed=1.0, max_motor_torque=1.0), xf, 0.0))
    for s in (-1e3, 1e3):
        j, xf = geo.place(FIXED, rng, coordinate=s)
        out.append((j, drive(0, S | L | M, lower=-2e3, upper=2e3, motor_speed=1.0, max_motor_torque=1.0), xf, 0.0))
    return out


def test_device_own_and_drive_rows_against_the_float64_geometry():
    cases = _poses()
    m = len(cases)
    s = _scene(2 * m)
    joints = np.zeros(m, nudge_b200.JOINT)
    drives = []
    grid = int(np.ceil(m ** (1.0 / 3.0)))
    for k, (j, d, xf, _) in enumerate(cases):
        a, b = 2 * k + 1, 2 * k + 2
        # each joint's pair moved to a cell of its own (the far ones stay where they are); a world anchor moves with it
        shift = np.zeros(3, np.float32) if np.abs(xf["position"]).max() > 1e3 else \
            np.float32(30.0) * np.array([k % grid, (k // grid) % grid + 20, k // (grid * grid)], np.float32)
        s.transforms[a] = xf[1]; s.transforms["position"][a] += shift
        s.transforms[b] = xf[2]; s.transforms["position"][b] += shift
        j = j.copy()
        j["a"] = a
        if int(j["b"]):
            j["b"] = b
        else:
            j["anchor_b"] = j["anchor_b"] + shift
        joints[k] = j
        if d is not None:
            d = d.copy(); d["joint"] = k
            drives.append(d)
    drives = np.array(drives, nudge_b200.JOINT_DRIVE)
    g = nudge_b200.Sim(s)
    g.upload_joints(joints); g.upload_joint_drives(drives)
    g.collide(); g.apply_gravity_damping(); g.read_cached_impulses(); g.setup_contact_constraints()
    rows = joint_rows(g)
    table = g.debug("joint_drives", dof.DRIVE_TABLE)
    g.download_bodies()
    order = joints_ref.table_order(joints)
    jt = joints[order]
    solve = rows[dof.solve_order(jt, table)]
    by_joint = {int(d["joint"]): d for d in drives}
    rng = np.random.default_rng(5)
    at, twist_worst = 0, 0.0
    for p, i in enumerate(order):
        count = joints_ref.ROWS_PER_TYPE[int(jt[p]["type"])] + dof.drive_row_count(int(table["flags"][p]))
        d = by_joint.get(int(i))
        twist_worst = max(twist_worst, check_joint(jt[p], d, g.transforms, solve[at:at + count], table[p] if d is not None else None, rng,
                                                   off=cases[i][3], dt=np.float32(s.time_step), where="joint %d" % i))
        at += count
    assert at == len(rows)
    assert twist_worst > 0.3


def _hinge_or_twist(typ, body, u, angle, lo, hi):
    """Body `body` (at its anchor, b the world) at the hinge angle or twist `angle` about the world axis u, with a [lo, hi] limit."""
    j = np.zeros(1, nudge_b200.JOINT)[0]
    j["type"], j["a"], j["b"], j["beta"] = typ, body, 0, 0.2
    j["axis_a"] = j["axis_b"] = u; j["rel_rotation"] = (0.0, 0.0, 0.0, 1.0)
    d = drive(0, L if typ == HINGE else TW, lower=lo, upper=hi)
    return j, d, Rotation.from_rotvec(-angle * np.asarray(u, np.float64)).as_quat()   # D = R_a turns b back onto a: theta = -a's angle


def test_wide_hinge_and_twist_ranges_do_not_brake_at_the_far_stop():
    """A hinge and a twist limit of [-3.1, 3.1] resting on the upper stop, turned away from it at 10 rad/s: the lower stop is 6.2 rad away,
    so its row stays at impulse 0 and the relative speed is still -10 rad/s after the step.  (With C = 2 sin((theta - lower) / 2) the lower
    row capped the speed at 2 sin(3.1) / dt = 5 rad/s.)"""
    s = _scene(2)
    u = np.array([0.0, 0.0, 1.0])
    joints, drives = [], []
    for k, typ in enumerate((HINGE, BALL)):
        body = k + 1
        s.transforms["position"][body] = (20.0 * k, 500.0, 0.0)
        j, d, q = _hinge_or_twist(typ, body, u, 3.1, -3.1, 3.1)
        j["anchor_b"] = s.transforms["position"][body]
        s.transforms["rotation"][body] = q
        s.momentum["angular_velocity"][body] = 10.0 * u   # d(theta)/dt = u . (0 - omega_a) = -10
        d["joint"] = k
        joints.append(j); drives.append(d)
    g = nudge_b200.Sim(s)
    g.upload_joints(np.array(joints)); g.upload_joint_drives(np.array(drives))
    g.download_bodies()
    before = [geo.coordinates(j, *geo.pose(g.transforms, k + 1), np.zeros(3), geo.IDENTITY) for k, j in enumerate(joints)]
    assert abs(before[0]["theta"] - 3.1) < 1e-5 and abs(before[1]["twist"] - 3.1) < 1e-5
    g.step_staged()
    g.download_bodies()
    back = g.download_joint_drives()
    for k in range(2):
        speed = -float(g.momentum["angular_velocity"][k + 1] @ u)
        assert back["impulse"][k][1] == 0.0, (k, back["impulse"][k])
        assert abs(speed + 10.0) < 1e-3, (k, speed)
        after = geo.coordinates(joints[k], *geo.pose(g.transforms, k + 1), np.zeros(3), geo.IDENTITY)
        a = after["theta"] if k == 0 else after["twist"]
        assert abs(a - (3.1 - 10.0 * float(s.time_step))) < 1e-3, (k, a)


def _pendulums():
    """Bodies hanging 0.5 below a joint to the world (a 0.2 x 0.9 x 0.2 box reaching to within 0.05 of it: a lever long against the body
    converges slowly, DESIGN.md section 8.20), each pushed into one limit, 30 apart: (scene, joints, drives, what each measures and
    its bounds).  Narrow ranges and ranges wider than pi, for hinge, twist, cone, slider and distance limits; plus a free hinge motor, a free
    slider motor and two blocked motors."""
    cases = [  # typ, flags, kwargs, velocity, angular velocity, measured coordinate
        (HINGE, L, dict(lower=-0.5, upper=0.5), (4.0, 0, 0), (0, 0, 0), "theta"),
        (HINGE, L, dict(lower=-3.0, upper=3.0), (9.0, 0, 0), (0, 0, 0), "theta"),
        (BALL, TW, dict(lower=-0.5, upper=0.5), (0, 0, 0), (0, 6.0, 0), "twist"),
        (BALL, TW, dict(lower=-3.0, upper=3.0), (0, 0, 0), (0, 12.0, 0), "twist"),
        (BALL, CN, dict(cone=0.5), (4.0, 0, 2.0), (0, 0, 0), "swing"),
        (BALL, CN, dict(cone=2.0), (9.0, 0, 3.0), (0, 0, 0), "swing"),
        (BALL, CN | TW, dict(cone=2.0, lower=-3.0, upper=3.0), (9.0, 0, 3.0), (0, 8.0, 0), "swing"),
        (FIXED, S | L, dict(lower=-0.3, upper=0.3), (0, 3.0, 0), (0, 0, 0), "s"),
        (FIXED, S | L, dict(lower=-3.0, upper=3.0), (0, 8.0, 0), (0, 0, 0), "s"),
        (DISTANCE, L, dict(lower=0.25, upper=0.5), (5.0, 0, 0), (0, 0, 0), "distance"),
        (HINGE, M, dict(motor_speed=2.0, max_motor_torque=100.0), (0, 0, 0), (0, 0, 0), "theta"),
        (FIXED, S | M, dict(motor_speed=1.5, max_motor_torque=100.0), (0, 0, 0), (0, 0, 0), "s"),
        (HINGE, L | M, dict(lower=-0.2, upper=0.2, motor_speed=3.0, max_motor_torque=2.0), (0, 0, 0), (0, 0, 0), "theta"),
        (HINGE, L | M, dict(lower=-0.2, upper=0.2, motor_speed=-3.0, max_motor_torque=2.0), (0, 0, 0), (0, 0, 0), "theta"),
    ]
    s = _scene(len(cases), size=0.1, gravity=9.82)
    s.box_data["size"][1:] = (0.1, 0.45, 0.1)
    s.properties[1:] = scenes._box_props(s.box_data["size"][1:])
    joints, drives = [], []
    for k, (typ, flags, kw, v, w, _) in enumerate(cases):
        body = k + 1
        o = np.array([30.0 * k, 500.0, 0.0], np.float32)
        j = np.zeros(1, nudge_b200.JOINT)[0]
        j["type"], j["a"], j["b"], j["beta"], j["rel_rotation"] = typ, body, 0, 0.2, (0.0, 0.0, 0.0, 1.0)
        if flags & S or flags & M and typ == HINGE:
            # a slider along the world axis (vertical for the stops, horizontal for the motor) and a vertical motor hinge: the body at its anchor
            axis = (0.0, 1.0, 0.0) if flags & L or typ == HINGE else (1.0, 0.0, 0.0)
            s.transforms["position"][body] = o
            j["anchor_b"] = o
        else:
            axis = (0.0, 0.0, 1.0) if typ == HINGE else (0.0, 1.0, 0.0)   # the hinge across the swing, the twist axis up to the anchor
            s.transforms["position"][body] = o - np.float32([0.0, 0.5, 0.0])
            j["anchor_a"], j["anchor_b"], j["length"] = (0.0, 0.5, 0.0), o, 0.5
            if typ == DISTANCE:
                j["anchor_a"] = (0.0, 0.0, 0.0)
        j["axis_a"] = j["axis_b"] = axis
        s.momentum["velocity"][body], s.momentum["angular_velocity"][body] = v, w
        d = drive(k, flags, **kw)
        joints.append(j); drives.append(d)
    return s, np.array(joints), np.array(drives), cases


def _coordinate(j, xf, key):
    c = geo.coordinates(j, *geo.pose(xf, int(j["a"])), np.zeros(3), geo.IDENTITY)
    return c[key]


def test_pendulums_stay_within_their_limits_and_motors_keep_the_header_sign():
    """300 graph replays with the coordinates measured in float64 from the downloaded transforms after every step.  Stated slack: 0.03
    rad past an angle stop, 0.01 past a slider or rope stop.  The free hinge motor turns b relative to a at +motor_speed within 1e-3 and the
    free slider motor moves s at +motor_speed within 1% (the header's signs); a motor blocked by a stop holds its impulse at +-max_motor_torque * dt,
    exactly."""
    s, joints, drives, cases = _pendulums()
    g = nudge_b200.Sim(s, stream=side_stream())
    g.upload_joints(joints); g.upload_joint_drives(drives)
    worst = np.zeros(len(cases))
    reached = np.zeros(len(cases))
    prev, rates = None, []
    dt = float(s.time_step)
    for step in range(300):
        g.step()
        g.download_bodies()
        assert np.isfinite(g.transforms["position"]).all()
        now = np.array([_coordinate(j, g.transforms, c[5]) for j, c in zip(joints, cases)])
        if prev is not None:
            rates.append((geo.wrap(now[10] - prev[10]) / dt, (now[11] - prev[11]) / dt))
        prev = now
        for k, (typ, flags, kw, *_rest) in enumerate(cases):
            if flags & CN:
                worst[k] = max(worst[k], now[k] - kw["cone"]); reached[k] = max(reached[k], now[k] - kw["cone"])
            elif flags & (L | TW):
                worst[k] = max(worst[k], now[k] - kw["upper"], kw["lower"] - now[k])
                reached[k] = max(reached[k], now[k] - kw["upper"], kw["lower"] - now[k])
    assert g.debug_scalar("graph_records") == 1
    print("worst past the stop:", dict(enumerate(np.round(worst, 5))))
    slack = np.array([0.03 if typ in (HINGE, BALL) else 0.01 for typ, *_ in cases])
    assert (worst < slack).all(), worst
    limited = [k for k, c in enumerate(cases) if c[1] & (L | CN | TW) and not c[1] & M]
    assert (reached[limited] > -0.05).all(), reached   # every pendulum reached its stop, so the bound was tested
    hinge_rate, slide_rate = np.array(rates[-30:]).T
    # the slider's lateral rows hold the body against gravity with a lever that grows with its travel (7.5 after 300 steps), which slows
    # their convergence (DESIGN.md section 8.20): its speed is held to 1%, the free hinge's to 1e-3
    assert np.abs(hinge_rate - 2.0).max() < 1e-3 and np.abs(slide_rate - 1.5).max() < 0.015, (hinge_rate[-3:], slide_rate[-3:])
    back = g.download_joint_drives()
    lim = np.float32(2.0) * np.float32(dt)
    assert back["impulse"][12][0] == lim and back["impulse"][13][0] == -lim, back["impulse"][12:]
