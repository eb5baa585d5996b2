"""The numpy restatement of the joint drives (tests/joint_drives_ref.py; DESIGN.md section 8.17) on the CPU: the nb_joint_drive layout against the
header, the half-angle conversion, and the restated rows solved by the host row loop (oracle/rows_ref.py): a hinge limit holds a pendulum, a
motor reaches its speed or, too weak, lets its load fall, a rope hangs at its length and pulls only when taut, and a joint breaks below its
steady load and never at twice it."""
import os
import subprocess
import numpy as np
import nudge_b200
from nudge_b200 import abi, scenes
from oracle import joints_ref, rows_ref
from tests import joint_drives_ref as drives_ref
from tests.test_joints_ref import _joint, _integrate

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DT = np.float32(1.0 / 60.0)
G = 9.81


def _drive(joint, flags, **kw):
    d = np.zeros(1, nudge_b200.JOINT_DRIVE)[0]
    d["joint"], d["flags"], d["break_force"], d["break_torque"] = joint, flags, np.inf, np.inf
    for k, v in kw.items():
        d[k] = v
    return d


def _run(joints, drives, xf, steps, gravity=True, sweeps=8, probe=None):
    """Steps bodies 0..len(xf)-1 (body 0 the world; unit mass, inertia 1/6 I, isotropic) with the restated rows: the break rule on the
    previous rows, the rows, the warm start and `sweeps` sweeps in solve order, then the integration.  probe(step, xf, lin, ang, rows, table)."""
    n = len(xf)
    lin, ang = np.zeros((n, 3)), np.zeros((n, 3))
    minv = np.array([0.0] + [1.0] * (n - 1))
    inv_i = np.stack([np.zeros((3, 3))] + [np.eye(3) * 6.0] * (n - 1))
    table, imp = drives_ref.drive_table(joints, drives)
    order = drives_ref.solve_order(joints, table)
    n_own = sum(joints_ref.ROWS_PER_TYPE[int(j["type"])] for j in joints)
    prev = None
    for step in range(steps):
        if gravity:
            lin[1:, 1] -= G * float(DT)
        if prev is not None:
            table["broken"] = drives_ref.broken_after(joints, prev, table, DT)
        rows = drives_ref.joint_rows(joints, xf, DT, table, imp)
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


def _pendulum(x=1.0):
    """Body 1 at (x, 0, 0), hinged to the world at the origin about z, unrotated at rest."""
    xf = np.zeros(2, scenes.TRANSFORM); xf["rotation"][:, 3] = 1.0
    xf["position"][1] = (x, 0.0, 0.0)
    j = _joint(joints_ref.HINGE, 1, 0, anchor_a=(-x, 0.0, 0.0), axis_a=(0.0, 0.0, 1.0), axis_b=(0.0, 0.0, 1.0))
    return xf, np.array([j])


def _theta(xf):
    """b's rotation relative to a about z: minus the pendulum's swing angle."""
    p = xf["position"][1].astype(np.float64)
    return -np.arctan2(p[1], p[0])


def test_drive_layout_matches_the_header(tmp_path):
    fields = nudge_b200.JOINT_DRIVE.names
    src = tmp_path / "layout.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "nudge_b200.h"\nint main(void) {\n' +
                   "".join('printf("%%zu\\n", offsetof(nb_joint_drive, %s));\n' % f for f in fields) +
                   'printf("%zu %d %d %d\\n", sizeof(nb_joint_drive), NB_JOINT_LIMIT, NB_JOINT_MOTOR, NB_JOINT_BREAKABLE); return 0; }\n')
    exe = tmp_path / "layout"
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), "-o", str(exe), str(src)])
    out = [int(x) for x in subprocess.check_output([str(exe)]).split()]
    assert out[:len(fields)] == [abi.JOINT_DRIVE.fields[f][1] for f in fields]
    assert out[len(fields):] == [56, drives_ref.LIMIT, drives_ref.MOTOR, drives_ref.BREAKABLE] and abi.JOINT_DRIVE.itemsize == 56
    assert (nudge_b200.JOINT_LIMIT, nudge_b200.JOINT_MOTOR, nudge_b200.JOINT_BREAKABLE) == (1, 2, 4)


def test_half_angles_are_within_one_ulp_of_float64():
    x = np.concatenate([np.linspace(-np.pi, np.pi, 4001), np.random.default_rng(1).uniform(-np.pi, np.pi, 4000)]).astype(np.float32)
    x = np.clip(x, np.float32(-np.pi), np.float32(np.pi))
    for i, fn in enumerate((np.sin, np.cos)):
        got = np.array([drives_ref.half_angle(v)[i] for v in x], np.float32).astype(np.float64)
        want = fn(0.5 * x.astype(np.float64))
        assert (np.abs(got - want) <= np.spacing(np.abs(want).astype(np.float32)).astype(np.float64)).all()


def test_rows_without_drives_are_todays_and_the_table_order_is_kept():
    xf, rng = np.zeros(4, scenes.TRANSFORM), np.random.default_rng(3)
    xf["rotation"][:, 3] = 1.0; xf["position"][1:] = rng.normal(size=(3, 3))
    joints = np.array([_joint(t, 1 + t % 3, (t + 1) % 4 if (t + 1) % 4 != 1 + t % 3 else 0, length=0.5) for t in range(4)])
    plain = drives_ref.joint_rows(joints, xf, DT)
    table = np.zeros(4, drives_ref.DRIVE_TABLE)
    assert drives_ref.joint_rows(joints, xf, DT, table).tobytes() == plain.tobytes()
    table, imp = drives_ref.drive_table(joints, np.array([_drive(1, 3, lower=-1.0, upper=1.0, impulse=(0.5, 0.25, 0.125)),
                                                          _drive(3, 1, lower=0.1, upper=2.0, impulse=(0.0, 1.0, 2.0))]))
    assert list(table["row"][[1, 3]]) == [0, 3] and list(imp) == [0.5, 0.25, 0.125, 1.0, 2.0]
    rows = drives_ref.joint_rows(joints, xf, DT, table, imp)
    assert len(rows) == 20
    for k in rows.dtype.names:
        if k not in ("lo", "hi"):
            assert rows[:15][k].tobytes() == plain[k].tobytes(), k
    assert rows[14]["lo"] == rows[14]["hi"] == 0 and list(rows["lo"][15:]) == [-rows["hi"][15], 0, 0, 0, 0]
    assert list(drives_ref.solve_order(joints, table)) == [0, 1, 2, 3, 4, 5, 6, 7, 15, 16, 17, 8, 9, 10, 11, 12, 13, 14, 18, 19]
    assert table["position"][3][0] > 0 and table["position"][1][1] > 0.99   # recorded in place


def test_a_hinge_limit_holds_a_pendulum():
    xf, joints = _pendulum()
    lo, hi = -0.3, 0.5
    seen = []
    table, lin, ang = _run(joints, np.array([_drive(0, drives_ref.LIMIT, lower=lo, upper=hi)]), xf, 240,
                           probe=lambda s, xf, *_: seen.append(_theta(xf)))
    assert max(seen) < hi + 0.02 and min(seen) > lo - 0.02, (min(seen), max(seen))
    assert abs(seen[-1] - hi) < 0.02                                            # it rests on the upper stop
    assert abs(2 * np.arctan2(table["position"][0][0], table["position"][0][1]) - seen[-2]) < 1e-3


def test_a_motor_with_ample_torque_reaches_its_speed():
    xf, joints = _pendulum(0.0)   # a wheel on its axle: anchor at the centre
    joints[0]["anchor_b"] = xf["position"][1]
    _, lin, ang = _run(joints, np.array([_drive(0, drives_ref.MOTOR, motor_speed=3.0, max_motor_torque=100.0)]), xf, 30, gravity=False)
    assert abs(-ang[1, 2] - 3.0) < 1e-3   # the hinge's relative speed u . (w_b - w_a), b the world


def test_a_motor_below_the_load_does_not_hold_it():
    """A horizontal arm: gravity's torque about the hinge is m g r = 9.81; a motor holding speed 0 keeps it up with 20, not with 5."""
    for torque, holds in ((20.0, True), (5.0, False)):
        xf, joints = _pendulum()
        seen = []
        _run(joints, np.array([_drive(0, drives_ref.MOTOR, motor_speed=0.0, max_motor_torque=torque)]), xf, 60, probe=lambda s, xf, *_: seen.append(_theta(xf)))
        assert (max(seen) < 0.05) == holds, (torque, max(seen))


def test_a_rope_hangs_at_its_length_and_pulls_only_when_taut():
    xf = np.zeros(2, scenes.TRANSFORM); xf["rotation"][:, 3] = 1.0
    xf["position"][1] = (0.0, -1.0, 0.0)
    joints = np.array([_joint(joints_ref.DISTANCE, 1, 0, length=1.0, anchor_b=(0.0, 0.0, 0.0))])
    L, slack_checked = 2.0, []

    def probe(step, xf, lin, ang, rows, table):
        dist = np.linalg.norm(xf["position"][1].astype(np.float64))
        assert rows["impulse"][0] == 0                                 # the own row stays in place
        if step < 200 and dist + np.linalg.norm(lin[1]) * float(DT) < L - 0.05:
            assert (rows["impulse"][1:] == 0).all(); slack_checked.append(step)
    _run(joints, np.array([_drive(0, drives_ref.LIMIT, lower=0.0, upper=L)]), xf, 300, probe=probe)
    assert len(slack_checked) > 10
    assert abs(np.linalg.norm(xf["position"][1].astype(np.float64)) - L) < 0.01


def test_a_joint_breaks_below_its_steady_load_and_never_above_twice_it():
    """A body hanging from a ball joint: the steady load is m g; a threshold of half breaks it, one of 2.5 times never does in 300 steps."""
    for force, breaks in ((0.5 * G, True), (2.5 * G, False)):
        xf = np.zeros(2, scenes.TRANSFORM); xf["rotation"][:, 3] = 1.0
        xf["position"][1] = (0.0, -1.0, 0.0)
        joints = np.array([_joint(joints_ref.BALL, 1, 0, anchor_a=(0.0, 1.0, 0.0), anchor_b=(0.0, 0.0, 0.0))])
        table, lin, _ = _run(joints, np.array([_drive(0, drives_ref.BREAKABLE, break_force=force)]), xf, 300)
        assert bool(table["broken"][0]) == breaks
        if breaks:
            assert xf["position"][1][1] < -10.0 and (joints["impulse"] == 0).all()   # it fell free
        else:
            assert abs(xf["position"][1][1] + 1.0) < 1e-3


def test_broken_rows_are_zero_rows_and_the_torque_rule_uses_angular_rows():
    xf, joints = _pendulum()
    table, imp = drives_ref.drive_table(joints, np.array([_drive(0, drives_ref.LIMIT | drives_ref.MOTOR | drives_ref.BREAKABLE, lower=-1.0, upper=1.0,
                                                                max_motor_torque=1.0, break_torque=1.0)]))
    rows = drives_ref.joint_rows(joints, xf, DT, table, imp)
    rows["impulse"] = 0; rows["impulse"][5] = np.float32(1.0 * DT) * 0.99   # the motor row: angular, just inside the torque threshold
    assert drives_ref.broken_after(joints, rows, table, DT)[0] == 0
    rows["impulse"][0] = 100.0                                                 # a linear row: the force threshold is +inf
    assert drives_ref.broken_after(joints, rows, table, DT)[0] == 0
    rows["impulse"][6] = np.float32(1.0 * DT) * 0.5                            # the lower limit row adds to A
    table["broken"] = drives_ref.broken_after(joints, rows, table, DT)
    assert table["broken"][0] == 1
    zero = drives_ref.joint_rows(joints, xf, DT, table, imp)
    assert (zero["a"] == 1).all() and (zero["b"] == 0).all()
    for k in zero.dtype.names:
        if k not in ("a", "b"):
            assert not np.frombuffer(zero[k].tobytes(), np.uint8).any(), k
