"""The numpy restatement of the joint springs (tests/joint_spring_ref.py; DESIGN.md section 8.21) on the CPU: the nb_joint_spring layout
against the header; the hinge target's half-angle conversion; without springs, joint_dof_ref's rows byte for byte; an initial error of
every spring coordinate shrinking under the host row loop (oracle/rows_ref.py), which pins the signs; single-body slider, hinge and distance
springs following the float64 backward-Euler recurrence; critical damping without overshoot; and a blocked spring at its force bound."""
import os
import subprocess
import numpy as np
import nudge_b200
from nudge_b200 import abi
from oracle import joints_ref, rows_ref
from tests import joint_dof_ref as dof
from tests import joint_spring_ref as spr
from tests.test_joints_ref import _joint, _integrate, _qmul
from tests.test_joint_dof_ref import _drive, _world, _random_old_set, _about

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DT = np.float32(1.0 / 60.0)
BALL, HINGE, FIXED, DISTANCE = joints_ref.BALL, joints_ref.HINGE, joints_ref.FIXED, joints_ref.DISTANCE
INERTIA = 1.0 / 6.0   # _run's bodies: unit mass, inertia I / 6


def spring(joint, target, stiffness, damping=0.0, target_velocity=0.0, max_force=np.inf, impulse=(0.0, 0.0, 0.0)):
    s = np.zeros(1, nudge_b200.JOINT_SPRING)[0]
    s["joint"], s["target_velocity"], s["stiffness"], s["damping"], s["max_force"], s["impulse"] = joint, target_velocity, stiffness, damping, max_force, impulse
    s["target"][:len(np.atleast_1d(target))] = target
    return s


def _run(joints, drives, springs, xf, steps, sweeps=8, probe=None, lin=None, ang=None):
    """Steps bodies 0..len(xf)-1 (body 0 the world) without gravity with the restated rows: the rows, the warm start and `sweeps` sweeps in
    solve order (own, spring, drive rows), then the integration.  probe(step, xf, lin, ang, spring_rows, spring_table)."""
    n = len(xf)
    lin = np.zeros((n, 3)) if lin is None else lin
    ang = np.zeros((n, 3)) if ang is None else ang
    minv = np.array([0.0] + [1.0] * (n - 1))
    inv_i = np.stack([np.zeros((3, 3))] + [np.eye(3) / INERTIA] * (n - 1))
    table, imp = dof.drive_table(joints, drives) if len(drives) else (None, None)
    stable, simp = spr.spring_table(joints, springs)
    order = spr.solve_order(joints, table, stable)
    n_own = sum(joints_ref.ROWS_PER_TYPE[int(j["type"])] for j in joints)
    for step in range(steps):
        rows, srows = spr.joint_rows(joints, xf, DT, table, imp, stable, simp)
        allr = np.concatenate([rows, srows])
        solve = allr[order]
        rows_ref.apply_rows(solve, lin, ang, minv, inv_i, warm=True)
        for _ in range(sweeps):
            rows_ref.apply_rows(solve, lin, ang, minv, inv_i)
        allr[order] = solve
        joints_ref.set_impulses(joints, allr[:n_own])
        if table is not None:
            imp = allr["impulse"][n_own:len(rows)].copy()
        simp = allr["impulse"][len(rows):].copy()
        _integrate(xf, lin, ang, float(DT))
        if probe:
            probe(step, xf, lin, ang, allr[len(rows):], stable)
    return stable, lin, ang


def _slider(start):
    """Body 1 at (start, 0, 0), welded to the world at the origin with x free (SLIDE), the anchor at its centre (on the axis): s = -x."""
    xf = _world()
    xf["position"][1] = (start, 0.0, 0.0)
    j = _joint(FIXED, 1, 0, anchor_a=(0.0, 0.0, 0.0), anchor_b=(0.0, 0.0, 0.0), axis_a=(1.0, 0.0, 0.0))
    return xf, np.array([j]), np.array([_drive(0, dof.SLIDE)])


def _hinge(angle):
    """Body 1 at the origin turned by `angle` about y, hinged to the world about y at its centre: theta = -angle."""
    xf = _world()
    xf["rotation"][1] = _about((0, 1, 0), angle)
    j = _joint(HINGE, 1, 0, anchor_a=(0.0, 0.0, 0.0), anchor_b=(0.0, 0.0, 0.0), axis_a=(0.0, 1.0, 0.0), axis_b=(0.0, 1.0, 0.0))
    return xf, np.array([j]), np.array([], nudge_b200.JOINT_DRIVE)


def _rope(length):
    """Body 1 at (0, -length, 0) on a distance joint of rest length 1 to the world origin."""
    xf = _world()
    xf["position"][1] = (0.0, -length, 0.0)
    j = _joint(DISTANCE, 1, 0, anchor_a=(0.0, 0.0, 0.0), anchor_b=(0.0, 0.0, 0.0), length=1.0)
    return xf, np.array([j]), np.array([], nudge_b200.JOINT_DRIVE)


def _coordinate(typ, xf):
    """The sprung coordinate in float64: s = -x, the hinge angle theta (minus body 1's angle about y), the distance."""
    if typ == FIXED:
        return -float(xf["position"][1][0])
    if typ == HINGE:
        q = xf["rotation"][1].astype(np.float64)
        return -2.0 * np.arctan2(q[1], q[3])
    return float(np.linalg.norm(xf["position"][1].astype(np.float64)))


def _recurrence(x0, target, k, c, m, steps, vt=0.0, dt=float(DT)):
    """Backward Euler of m x'' = -k (x - target) - c (x' - vt) in float64, from rest: v' = (m v - dt (k (x - target) - c vt)) / (m + dt c +
    dt^2 k), x' = x + dt v'."""
    x, v, out = x0, 0.0, []
    for _ in range(steps):
        v = (m * v - dt * (k * (x - target) - c * vt)) / (m + dt * c + dt * dt * k)
        x = x + dt * v
        out.append(x)
    return np.array(out)


def test_spring_layout_matches_the_header(tmp_path):
    fields = nudge_b200.JOINT_SPRING.names
    assert nudge_b200.JOINT_SPRING is abi.JOINT_SPRING
    src = tmp_path / "layout.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "nudge_b200.h"\nint main(void) {\n' +
                   "".join('printf("%%zu\\n", offsetof(nb_joint_spring, %s));\n' % f for f in fields) +
                   'printf("%zu\\n", sizeof(nb_joint_spring)); return 0; }\n')
    exe = tmp_path / "layout"
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), "-o", str(exe), str(src)])
    out = [int(x) for x in subprocess.check_output([str(exe)]).split()]
    assert out == [abi.JOINT_SPRING.fields[f][1] for f in fields] + [56]


def test_hinge_target_half_angles_are_within_one_ulp_of_float64():
    x = np.concatenate([np.linspace(-np.pi, np.pi, 4001), np.random.default_rng(2).uniform(-np.pi, np.pi, 4000)]).astype(np.float32)
    x = np.clip(x, np.float32(-np.pi), np.float32(np.pi))
    joints = _hinge(0.0)[1]
    for v in x[::8]:
        table, _ = spr.spring_table(joints, [spring(0, v, 1.0)])
        got = table["target"][0][:2].astype(np.float64)
        want = np.array([np.sin(0.5 * np.float64(v)), np.cos(0.5 * np.float64(v))])
        assert (np.abs(got - want) <= np.spacing(np.abs(want).astype(np.float32)).astype(np.float64)).all(), v
        assert table["angle"][0] == v and (table["target"][0][2:] == 0).all()


def test_without_springs_the_rows_are_joint_dof_refs():
    joints, drives, xf = _random_old_set(11)
    table, imp = dof.drive_table(joints, drives)
    want = dof.joint_rows(joints, xf.copy(), DT, table.copy(), imp)
    for springs in (None, np.zeros(len(joints), spr.SPRING_TABLE)):
        rows, srows = spr.joint_rows(joints, xf.copy(), DT, table.copy(), imp, springs)
        assert rows.tobytes() == want.tobytes() and len(srows) == 0
    assert (spr.solve_order(joints, table, None) == dof.solve_order(joints, table)).all()


def test_an_initial_error_of_every_spring_coordinate_shrinks():
    """Each type from an offset start toward its target under a damped spring; the ball's target is a rotation 0.5 rad away."""
    cases = [(FIXED, _slider(0.0), 0.5), (HINGE, _hinge(0.0), 0.5), (DISTANCE, _rope(1.0), 1.5), (HINGE, _hinge(0.3), -2.5)]
    for typ, (xf, joints, drives), target in cases:
        x0 = _coordinate(typ, xf)
        _run(joints, drives, [spring(0, target, 20.0, 2.0)], xf, 120)
        assert abs(_coordinate(typ, xf) - target) < 0.05 * abs(x0 - target), (typ, target)
    xf = _world()
    joints = np.array([_joint(BALL, 1, 0, anchor_a=(0.0, 0.0, 0.0), anchor_b=(0.0, 0.0, 0.0))])
    axis = np.array([1.0, 2.0, -0.5]) / np.linalg.norm([1.0, 2.0, -0.5])
    target = _about(axis, 0.5).astype(np.float32)
    table, _, _ = _run(joints, [], [spring(0, target, 20.0, 2.0)], xf, 120)
    # conj(q_a) * q_b with b the world is conj(q_a): the ball settles where qmul(q_a, target) is the identity
    d = _qmul(xf["rotation"][1].astype(np.float64), target.astype(np.float64))
    assert 2.0 * np.arctan2(np.linalg.norm(d[:3]), abs(d[3])) < 0.025
    assert abs(spr.spring_position(BALL, table["position"][0])) < 0.025


def test_a_hinge_spring_across_the_seam_goes_the_long_way():
    """theta = -3.0 and a target of +3.0: the spring turns the hinge up through 0 to the target and never across -pi, as a LIMIT of
    [-pi, pi] lets the hinge turn (C = m(theta - target) is increasing over the whole difference, not wrapped)."""
    xf, joints, drives = _hinge(3.0)   # theta = -3.0
    k = 20.0
    got = []
    _run(joints, drives, [spring(0, 3.0, k, 2.0 * np.sqrt(k * INERTIA))], xf, 600, probe=lambda step, xf, *_: got.append(_coordinate(HINGE, xf)))
    got = np.array(got)
    # the angle as measured does not wrap at +-pi (it is twice a half angle), so a turn across the seam would read below -3.0
    assert got[0] > -3.0 and (np.diff(got) > -1e-6).all()   # critically damped: up all the way
    assert (got > 0.0).any() and (got < -2.5).any()
    assert abs(got[-1] - 3.0) < 0.01


def test_single_body_springs_follow_the_backward_euler_recurrence():
    """No gravity, no damping, the anchor on the axis: one spring row on one body, whose other rows act across it, so one sweep gives the
    implicit step exactly; 600 steps of float32 state against the float64 recurrence."""
    for typ, (xf, joints, drives), target, k, c, m in ((FIXED, _slider(-0.4), 0.1, 30.0, 0.0, 1.0), (FIXED, _slider(0.3), -0.2, 50.0, 1.5, 1.0),
                                                        (HINGE, _hinge(0.05), 0.02, 2.0, 0.0, INERTIA), (DISTANCE, _rope(1.6), 1.2, 40.0, 0.0, 1.0)):
        x0 = _coordinate(typ, xf)
        want = _recurrence(x0, target, k, c, m, 600)
        got = []
        _run(joints, drives, [spring(0, target, k, c)], xf, 600, probe=lambda step, xf, *_: got.append(_coordinate(typ, xf)))
        amp = abs(x0 - target)
        # float32 positions over 600 steps; the hinge's C = 2 sin((theta - target) / 2) and its first-order rotation update differ from
        # the linear recurrence at third order in the 0.03 rad amplitude
        tol = 2e-3 * amp if typ == HINGE else 2e-4 * amp + 2e-6
        assert np.abs(np.array(got) - want).max() < tol, (typ, np.abs(np.array(got) - want).max(), tol)
        assert abs(min(got) - target) > 0.5 * amp or abs(max(got) - target) > 0.5 * amp   # it oscillates (c = 0) or decays


def test_critical_damping_does_not_overshoot():
    k = 40.0
    xf, joints, drives = _slider(-1.0)
    got = []
    _run(joints, drives, [spring(0, 0.0, k, 2.0 * np.sqrt(k))], xf, 300, probe=lambda step, xf, *_: got.append(_coordinate(FIXED, xf)))
    got = np.array(got)
    assert (got <= 1.0 + 1e-6).all() and (got >= -1e-6).all() and (np.diff(got) <= 1e-7).all() and got[-1] < 1e-3


def test_a_blocked_spring_holds_exactly_its_force_bound():
    """A stiff slider spring pulled past the slider's upper stop: the stop holds the body, the spring row sits at max_force * dt."""
    xf, joints, drives = _slider(0.0)
    drives["flags"] = dof.SLIDE | dof.LIMIT
    drives["lower"], drives["upper"] = -1.0, 0.2
    impulses = []
    for target, sign in ((5.0, -1.0), (-5.0, 1.0)):
        xf, joints, _ = _slider(0.0)
        d = drives.copy()
        if sign > 0:
            d["lower"], d["upper"] = -0.2, 1.0
        _run(joints, d, [spring(0, target, 1000.0, 10.0, max_force=3.0)], xf, 120, probe=lambda step, xf, lin, ang, sr, st: impulses.append(sr["impulse"][0]))
        bound = np.float32(np.float32(3.0) * DT)
        # the spring row's Jacobian is J_s, on s: its impulse pushes s toward the target, so its sign is the target's side
        assert impulses[-1] == (bound if target > 0 else -bound), impulses[-1]
        assert abs(_coordinate(FIXED, xf) - (0.2 if target > 0 else -0.2)) < 0.02
