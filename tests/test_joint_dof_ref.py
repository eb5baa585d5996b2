"""The numpy restatement of sliders and swing-twist limits (tests/joint_dof_ref.py; DESIGN.md section 8.20) on the CPU: the nb_joint_drive
layout and flag values against the header; the cone's half-angle conversion; the swing-twist split; for the drive flags that existed
before, the same rows, table and break flags as tests/joint_drives_ref.py; an initial violation of every new row shrinking under the host
row loop (oracle/rows_ref.py), which pins the signs; and sliders, cones and twist limits holding bodies, with the break rule's force and
torque classes."""
import hashlib
import os
import subprocess
import numpy as np
import nudge_b200
from nudge_b200 import abi, scenes
from oracle import joints_ref, rows_ref
from tests import joint_dof_ref as dof
from tests import joint_drives_ref as drives_ref
from tests.test_joints_ref import _joint, _integrate, _qmul
from tests.test_gpu_rows import _quat_rotate

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DT = np.float32(1.0 / 60.0)
G = 9.81
L, M, BR = dof.LIMIT, dof.MOTOR, dof.BREAKABLE
S, CN, TW = dof.SLIDE, dof.CONE, dof.TWIST


def _drive(joint, flags, **kw):
    d = np.zeros(1, nudge_b200.JOINT_DRIVE)[0]
    d["joint"], d["flags"], d["break_force"], d["break_torque"] = joint, flags, np.inf, np.inf
    for k, v in kw.items():
        d[k] = v
    return d


def _run(joints, drives, xf, steps, gravity=True, sweeps=8, probe=None, lin=None, ang=None):
    """Steps bodies 0..len(xf)-1 (body 0 the world; unit mass, inertia 1/6 I) with the restated rows: the break rule on the previous rows,
    the rows, the warm start and `sweeps` sweeps in solve order, then the integration.  probe(step, xf, lin, ang, rows, table)."""
    n = len(xf)
    lin = np.zeros((n, 3)) if lin is None else lin
    ang = np.zeros((n, 3)) if ang is None else ang
    minv = np.array([0.0] + [1.0] * (n - 1))
    inv_i = np.stack([np.zeros((3, 3))] + [np.eye(3) * 6.0] * (n - 1))
    table, imp = dof.drive_table(joints, drives)
    order = dof.solve_order(joints, table)
    n_own = sum(joints_ref.ROWS_PER_TYPE[int(j["type"])] for j in joints)
    prev = None
    for step in range(steps):
        if gravity:
            lin[1:, 1] -= G * float(DT)
        if prev is not None:
            table["broken"] = dof.broken_after(joints, prev, table, DT)
        rows = dof.joint_rows(joints, xf, DT, table, imp)
        solve = rows[order]
        rows_ref.apply_rows(solve, lin, ang, minv, inv_i, warm=True)
        for _ in range(sweeps):
            rows_ref.apply_rows(solve, lin, ang, minv, inv_i)
        rows[order] = solve
        joints_ref.set_impulses(joints, rows[:n_own]); imp = rows["impulse"][n_own:].copy()
        prev = rows
        _integrate(xf, lin, ang, float(DT))
        if probe:
            probe(step, xf, lin, ang, rows, table)
    return table, lin, ang


def _world(n=2):
    xf = np.zeros(n, scenes.TRANSFORM); xf["rotation"][:, 3] = 1.0
    return xf


def _slider(axis, start=(0.0, 0.0, 0.0)):
    """Body 1 at `start`, welded to the world at the origin with its translation along `axis` (unit, world = body frame at rest) free."""
    xf = _world()
    xf["position"][1] = start
    j = _joint(joints_ref.FIXED, 1, 0, anchor_a=(0.0, 0.0, 0.0), anchor_b=(0.0, 0.0, 0.0), axis_a=axis)
    return xf, np.array([j])


def _s(xf, axis):
    """The slider coordinate s = dot(wb - wa, u) in float64 (b the world at the origin, the anchor at the body's centre)."""
    return -float(xf["position"][1].astype(np.float64) @ _quat_rotate(xf["rotation"][1].astype(np.float64), np.asarray(axis, np.float64)))


def _hanging(axis=(0.0, 1.0, 0.0)):
    """Body 1 hanging 1 below a ball joint to the world at the origin; axis_a (the twist axis) points from the body up to the anchor."""
    xf = _world()
    xf["position"][1] = (0.0, -1.0, 0.0)
    j = _joint(joints_ref.BALL, 1, 0, anchor_a=(0.0, 1.0, 0.0), anchor_b=(0.0, 0.0, 0.0), axis_a=axis)
    return xf, np.array([j])


def _swing_twist64(q, axis):
    """(swing, twist) in float64 of body a's rotation q against the world (rel_rotation identity), as the header's split measures them."""
    q = np.asarray(q, np.float64)
    q = -q if q[3] < 0 else q
    u = _quat_rotate(q, np.asarray(axis, np.float64))
    a_ = q[:3] @ u
    p = q[:3] - u * a_
    return 2.0 * np.arctan2(np.linalg.norm(p), np.hypot(a_, q[3])), 2.0 * np.arctan2(-a_, q[3])


def _about(axis, angle):
    axis = np.asarray(axis, np.float64) / np.linalg.norm(axis)
    return np.append(np.sin(0.5 * angle) * axis, np.cos(0.5 * angle))


def test_drive_layout_cone_and_new_flags_match_the_header(tmp_path):
    fields = nudge_b200.JOINT_DRIVE.names
    assert fields[-1] == "cone" and abi.JOINT_DRIVE.fields["cone"][0] == np.float32
    src = tmp_path / "layout.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "nudge_b200.h"\nint main(void) {\n' +
                   "".join('printf("%%zu\\n", offsetof(nb_joint_drive, %s));\n' % f for f in fields) +
                   'printf("%zu %zu %d %d %d\\n", sizeof(nb_joint_drive), sizeof(nb_joint), NB_JOINT_SLIDE, NB_JOINT_CONE, NB_JOINT_TWIST);\n'
                   'nb_joint_drive d; d.cone = 0.5f; printf("%d\\n", (int)(d.cone * 4.0f)); return 0; }\n')
    exe = tmp_path / "layout"
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), "-o", str(exe), str(src)])
    out = [int(x) for x in subprocess.check_output([str(exe)]).split()]
    assert out[:len(fields)] == [abi.JOINT_DRIVE.fields[f][1] for f in fields]
    assert out[len(fields):] == [56, 112, S, CN, TW, 2]   # cone is a float
    assert (nudge_b200.JOINT_SLIDE, nudge_b200.JOINT_CONE, nudge_b200.JOINT_TWIST) == (16, 32, 64)
    assert dof.DRIVE_TABLE.names[-1] == "cone" and dof.DRIVE_TABLE.fields["cone"][1] == 60


def test_cone_half_angles_are_within_one_ulp_of_float64():
    x = np.concatenate([np.linspace(1e-4, np.pi, 4001), np.random.default_rng(2).uniform(0.0, np.pi, 4000)]).astype(np.float32)
    x = np.clip(x, np.float32(1e-6), np.float32(np.pi))
    xf, joints = _hanging()
    for i, fn in enumerate((np.sin, np.cos)):
        got = np.array([dof.drive_table(joints, [_drive(0, CN, cone=v)])[0][("motor_speed", "max_motor_torque")[i]][0] for v in x[::16]], np.float64)
        want = fn(0.5 * x[::16].astype(np.float64))
        assert (np.abs(got - want) <= np.spacing(np.abs(want).astype(np.float32)).astype(np.float64)).all()
    table, _ = dof.drive_table(joints, [_drive(0, CN, cone=np.float32(0.7))])
    assert table["cone"][0] == np.float32(0.7)


def test_swing_twist_split():
    """ss^2 + cs^2 = 1 to float32 rounding; a pure twist and a pure swing come back as float64 angles within 2e-6 rad."""
    rng = np.random.default_rng(5)
    f = np.float32
    for q in scenes._random_unit_quaternions(rng, 500):
        axis = rng.normal(size=3); axis /= np.linalg.norm(axis)
        u = joints_ref.qrot(joints_ref._v(q), joints_ref._v(axis))
        p, ss, cs, st, ct = dof.swing_twist(tuple(f(x) for x in (-q if q[3] < 0 else q)), u)
        assert abs(float(ss) ** 2 + float(cs) ** 2 - 1.0) < 4e-6 and abs(float(st) ** 2 + float(ct) ** 2 - 1.0) < 4e-6
    u = (f(0.0), f(1.0), f(0.0))
    for angle in np.linspace(-3.0, 3.0, 61):
        _, ss, cs, st, ct = dof.swing_twist(tuple(f(x) for x in _about((0, 1, 0), angle)), u)   # d = q_a: twist = minus a's angle
        assert abs(2 * np.arctan2(float(st), float(ct)) + angle) < 2e-6 and float(ss) < 1e-7
        perp = (np.cos(angle), 0.0, np.sin(angle))
        _, ss, cs, st, ct = dof.swing_twist(tuple(f(x) for x in _about(perp, abs(angle))), u)
        assert abs(2 * np.arctan2(float(ss), float(cs)) - abs(angle)) < 2e-6 and float(st) == 0.0


def _random_old_set(seed):
    """Random joints of every type with random drives of the flags that existed before SLIDE, CONE and TWIST, some broken; and transforms."""
    rng = np.random.default_rng(seed)
    n, m = 12, 60
    xf = _world(n + 1)
    xf["position"][1:] = rng.normal(size=(n, 3)) * 2.0
    xf["rotation"][1:] = scenes._random_unit_quaternions(rng, n)
    joints = np.zeros(m, nudge_b200.JOINT)
    joints["type"] = rng.integers(0, 4, m); joints["a"] = rng.integers(1, n + 1, m); joints["b"] = rng.integers(0, n + 1, m)
    same = joints["a"] == joints["b"]; joints["b"][same] = joints["a"][same] % n + 1
    for k in ("anchor_a", "anchor_b"):
        joints[k] = rng.normal(size=(m, 3))
    for k in ("axis_a", "axis_b"):
        v = rng.normal(size=(m, 3)); joints[k] = v / np.linalg.norm(v, axis=1, keepdims=True)
    joints["rel_rotation"] = scenes._random_unit_quaternions(rng, m)
    joints["length"] = rng.random(m) * 3.0; joints["beta"] = 0.1 + 0.2 * rng.random(m); joints["softness"] = np.where(rng.random(m) < 0.5, 0.01, 0.0)
    joints["impulse"] = rng.normal(size=(m, 6)) * 0.1
    takes = {0: BR, 1: L | M | BR, 2: BR, 3: L | BR}
    drives, seen = [], [0, 0, 0, 0]
    for i in range(m):
        if i % 5:   # each type's drives cycle through every flag combination it takes
            t = int(joints[i]["type"])
            lo, hi = np.sort(rng.uniform(-np.pi, np.pi, 2)) if t == 1 else np.sort(rng.uniform(0.0, 3.0, 2))
            seen[t] += 1
            drives.append(_drive(i, seen[t] % 8 & takes[t], lower=lo, upper=hi, motor_speed=rng.normal(), max_motor_torque=rng.random() * 5,
                                 break_force=rng.random() * 5, break_torque=rng.random() * 5, impulse=rng.normal(size=3) * 0.1,
                                 broken=int(rng.random() < 0.1)))
    return joints, np.array(drives), xf


# sha256 of the bytes tests/joint_drives_ref.py gave for _random_old_set(11) before SLIDE, CONE and TWIST existed: the table, the first
# build's rows, the break flags on those rows and the solve order; recorded again when the angle limit measure stopped folding back past a
# half turn (DESIGN.md section 8.17), which changed the bias of six hinge limit rows and nothing else, and again when the drive rows got a
# buffer of their own, which lowered each driven entry's row by the 214 own rows and changed nothing else
OLD_DIGEST = "b4e7bd8a08829f2637ffe4e11d2a815584c92de646846c6235f2e9b3f0c0aef7"


def _old_bytes(ref, joints, drives, xf):
    table, imp = ref.drive_table(joints, drives)
    rows = ref.joint_rows(joints, xf, DT, table, imp)
    rows["impulse"] = np.random.default_rng(1).normal(size=len(rows)).astype(np.float32) * 0.2
    return table.tobytes() + rows.tobytes() + ref.broken_after(joints, rows, table, DT).tobytes() + ref.solve_order(joints, table).tobytes()


def test_drives_without_the_new_flags_are_unchanged():
    joints, drives, xf = _random_old_set(11)
    assert len({int(d["flags"]) for d in drives}) == 8
    want = _old_bytes(drives_ref, joints, drives, xf.copy())
    assert hashlib.sha256(want).hexdigest() == OLD_DIGEST
    assert _old_bytes(dof, joints, drives, xf.copy()) == want
    assert dof.joint_rows(joints, xf, DT).tobytes() == drives_ref.joint_rows(joints, xf, DT).tobytes()
    for fl in range(8):
        assert dof.drive_row_count(fl) == drives_ref.drive_row_count(fl)


def _decays(joints, drives, xf, measure, steps=120, **kw):
    e0 = measure(xf)
    _run(joints, drives, xf, steps, gravity=False, **kw)
    return e0, measure(xf)


def test_an_initial_violation_of_every_new_row_shrinks():
    """Each starts violated with the bodies at rest: the slider's drift across its axis, its lower and its upper stop, the cone and both
    twist stops.  Solved and integrated without gravity, each violation must fall below 2% of its start; this pins every new row's sign."""
    axis = np.array([0.6, 0.8, 0.0], np.float32)
    u = axis.astype(np.float64)

    def drift(xf):
        p = xf["position"][1].astype(np.float64)
        return np.linalg.norm(p - (p @ u) * u)
    xf, joints = _slider(axis, start=(0.4, -0.3, 0.25))
    e0, e1 = _decays(joints, [_drive(0, S)], xf, drift)
    assert e0 > 0.4 and e1 < 0.02 * e0, (e0, e1)
    # a stop row only pushes: the body leaves the violated stop with the speed the correction gave it, so the measure is how far the
    # coordinate lies outside its range
    def outside(x, lo, hi):
        return max(lo - x, x - hi, 0.0)
    for start in (1.5, -1.5):   # s = -start: past the lower stop, then past the upper one
        xf, joints = _slider(axis, start=tuple(start * axis))
        e0, e1 = _decays(joints, [_drive(0, S | L, lower=-1.0, upper=1.0)], xf, lambda xf: outside(_s(xf, axis), -1.0, 1.0))
        assert e0 > 0.4 and e1 < 0.02 * e0, (start, e0, e1)
    xf, joints = _hanging()
    xf["rotation"][1] = _about((1.0, 0.0, 0.3), 0.9)
    e0, e1 = _decays(joints, [_drive(0, CN, cone=0.5)], xf, lambda xf: outside(_swing_twist64(xf["rotation"][1], (0, 1, 0))[0], 0.0, 0.5))
    assert e0 > 0.3 and e1 < 0.02 * e0, (e0, e1)
    for angle in (0.9, -0.9):   # a's rotation about u by angle: twist = -angle
        xf, joints = _hanging()
        xf["rotation"][1] = _about((0.0, 1.0, 0.0), angle)
        e0, e1 = _decays(joints, [_drive(0, TW, lower=-0.4, upper=0.4)], xf, lambda xf: outside(_swing_twist64(xf["rotation"][1], (0, 1, 0))[1], -0.4, 0.4))
        assert e0 > 0.4 and e1 < 0.02 * e0, (angle, e0, e1)


def test_a_tilted_slider_under_gravity_slides_and_stays_on_its_line():
    axis = np.array([0.6, 0.8, 0.0], np.float32)
    u = axis.astype(np.float64)
    xf, joints = _slider(axis)
    off = []
    _, lin, ang = _run(joints, [_drive(0, S)], xf, 120, probe=lambda s, xf, *_: off.append(
        np.linalg.norm(xf["position"][1].astype(np.float64) - (xf["position"][1].astype(np.float64) @ u) * u)))
    t = 120 * float(DT)
    want = -0.5 * G * 0.8 * t * t   # the along-axis share of gravity, 0.8 g
    got = float(xf["position"][1].astype(np.float64) @ u)
    assert abs(got - want) < 0.03 * abs(want), (got, want)
    # the lateral rows' lever arm grows with the travel (about 15 here), which slows the sweeps' convergence: 0.2% of the travel
    assert max(off) < 2e-3 * abs(want) and abs(xf["rotation"][1][3] - 1.0) < 1e-5, (max(off), xf["rotation"][1])


def test_a_vertical_slider_rests_on_its_stop():
    xf, joints = _slider((0.0, 1.0, 0.0))   # s = -y: the body falls with s growing; the upper stop at 1 catches it
    seen = []
    _run(joints, [_drive(0, S | L, lower=-2.0, upper=1.0)], xf, 240, probe=lambda s, xf, *_: seen.append(_s(xf, (0, 1, 0))))
    assert max(seen) < 1.0 + 0.01 and abs(seen[-1] - 1.0) < 0.01 and seen[30] > 0.9


def test_a_slider_motor_reaches_its_speed_and_a_weak_one_sags():
    xf, joints = _slider((1.0, 0.0, 0.0))
    _, lin, _ = _run(joints, [_drive(0, S | M, motor_speed=2.0, max_motor_torque=100.0)], xf, 30, gravity=False)
    assert abs(-lin[1, 0] - 2.0) < 1e-3                # ds/dt = -dot(v_a, u)
    for force, holds in ((20.0, True), (5.0, False)):   # a vertical slider holding speed 0 against m g = 9.81
        xf, joints = _slider((0.0, 1.0, 0.0))
        _run(joints, [_drive(0, S | M, motor_speed=0.0, max_motor_torque=force)], xf, 60)
        assert (abs(float(xf["position"][1][1])) < 0.01) == holds, (force, xf["position"][1])


def test_a_pendulum_on_a_30_degree_cone_never_leaves_it():
    """Released at the bottom with 4 m/s sideways (enough to swing past 70 degrees freely), over 300 steps the swing stays within 0.03 rad of
    the cone."""
    cone = np.radians(30.0)
    xf, joints = _hanging()
    lin = np.zeros((2, 3)); lin[1] = (4.0, 0.0, 0.0)
    seen = []
    table, _, _ = _run(joints, [_drive(0, CN, cone=cone)], xf, 300, lin=lin,
                       probe=lambda s, xf, *_: seen.append(np.arccos(-xf["position"][1].astype(np.float64)[1] / np.linalg.norm(xf["position"][1]))))
    assert max(seen) < cone + 0.03 and max(seen) > cone - 0.05, max(seen)
    assert abs(2 * np.arctan2(float(table["position"][0][0]), float(table["position"][0][1])) - seen[-2]) < 0.01


def test_a_twist_limit_stops_a_spun_body():
    xf, joints = _hanging()
    ang = np.zeros((2, 3)); ang[1] = (0.0, 6.0, 0.0)
    seen = []
    _run(joints, [_drive(0, TW | CN, lower=-0.5, upper=0.5, cone=0.3)], xf, 200, ang=ang,
         probe=lambda s, xf, *_: seen.append(_swing_twist64(xf["rotation"][1], (0, 1, 0))[1]))
    assert min(seen) > -0.5 - 0.03 and abs(seen[-1] + 0.5) < 0.03, (min(seen), seen[-1])   # spun positively, the twist (minus it) stops at -0.5


def test_the_break_rule_counts_slider_limits_as_force_and_cones_as_torque():
    xf, joints = _slider((1.0, 0.0, 0.0))
    for force, torque, breaks in ((1.0, np.inf, True), (np.inf, 1.0, False)):
        table, imp = dof.drive_table(joints, [_drive(0, S | L | BR, lower=-1.0, upper=1.0, break_force=force, break_torque=torque)])
        rows = dof.joint_rows(joints, xf, DT, table, imp)
        rows["impulse"] = 0; rows["impulse"][7] = np.float32(2.0 * DT)   # the lower limit row
        assert dof.broken_after(joints, rows, table, DT)[0] == breaks
    xf, joints = _hanging()
    for force, torque, breaks in ((1.0, np.inf, False), (np.inf, 1.0, True)):
        table, imp = dof.drive_table(joints, [_drive(0, CN | TW | BR, lower=-1.0, upper=1.0, cone=0.5, break_force=force, break_torque=torque)])
        rows = dof.joint_rows(joints, xf, DT, table, imp)
        rows["impulse"] = 0; rows["impulse"][3] = np.float32(2.0 * DT)   # the cone row
        assert dof.broken_after(joints, rows, table, DT)[0] == breaks
        table["broken"] = 1
        zero = dof.joint_rows(joints, xf, DT, table, imp)
        assert len(zero) == 6 and not np.frombuffer(zero["lin_a"].tobytes() + zero["ang_b"].tobytes() + zero["bias"].tobytes(), np.uint8).any()
