"""The numpy restatement of the joints' row construction (oracle/joints_ref.py) on the CPU: BALL rows against the ball-joint helper of the row
tests, the bias signs of every type (an initial error must shrink under the row solver), the level assignment, and the nb_joint layout of
nudge_b200/abi.py against the header."""
import os
import subprocess
import numpy as np
import nudge_b200
from nudge_b200 import abi, scenes
from oracle import joints_ref, rows_ref
from tests.test_gpu_rows import ball_joint_rows, _quat_rotate

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _joint(type_, a, b, **kw):
    j = np.zeros(1, nudge_b200.JOINT)[0]
    j["type"], j["a"], j["b"], j["beta"] = type_, a, b, 0.2
    j["axis_a"] = j["axis_b"] = (0.0, 1.0, 0.0); j["rel_rotation"] = (0.0, 0.0, 0.0, 1.0)
    for k, v in kw.items():
        j[k] = v
    return j


def _transforms(n, seed):
    rng = np.random.default_rng(seed)
    xf = np.zeros(n, scenes.TRANSFORM)
    xf["rotation"][:, 3] = 1.0
    xf["position"][1:] = rng.normal(size=(n - 1, 3)) * 3.0
    xf["rotation"][1:] = scenes._random_unit_quaternions(rng, n - 1)
    return xf, rng


def test_ball_rows_equal_the_ball_joint_helper():
    xf, rng = _transforms(9, 1)
    for a, b in ((1, 0), (2, 3), (8, 4)):
        aa, ab = rng.normal(size=3), rng.normal(size=3)
        j = _joint(joints_ref.BALL, a, b, anchor_a=aa, anchor_b=ab)
        got = joints_ref.joint_rows([j], xf, 1.0 / 60.0)
        want = ball_joint_rows(xf, a, b, j["anchor_a"], j["anchor_b"], 1.0 / 60.0)
        assert len(got) == 3
        for k in ("lin_a", "ang_a", "lin_b", "ang_b", "bias"):
            np.testing.assert_allclose(got[k], want[k], rtol=0, atol=3e-5 * max(1.0, np.abs(want[k]).max()), err_msg=k)
        for k in ("a", "b", "lo", "hi"):
            assert (got[k] == want[k]).all()


def _qmul(l, r):
    return np.append(l[3] * r[:3] + r[3] * l[:3] + np.cross(l[:3], r[:3]), l[3] * r[3] - l[:3] @ r[:3])


def _errors(j, xf):
    """The position and angular error of joint j in float64, by the geometry (not by the rows)."""
    a, b = int(j["a"]), int(j["b"])
    pa, qa = xf["position"][a].astype(np.float64), xf["rotation"][a].astype(np.float64)
    pb, qb = xf["position"][b].astype(np.float64), xf["rotation"][b].astype(np.float64)
    wa = pa + _quat_rotate(qa, j["anchor_a"].astype(np.float64))
    wb = pb + _quat_rotate(qb, j["anchor_b"].astype(np.float64)) if b else j["anchor_b"].astype(np.float64)
    t = int(j["type"])
    if t == joints_ref.DISTANCE:
        return abs(np.linalg.norm(wa - wb) - float(j["length"])), 0.0
    ang = 0.0
    if t == joints_ref.HINGE:
        u = _quat_rotate(qa, j["axis_a"].astype(np.float64)); w = _quat_rotate(qb, j["axis_b"].astype(np.float64)) if b else j["axis_b"].astype(np.float64)
        ang = np.linalg.norm(np.cross(u, w))
    if t == joints_ref.FIXED:
        d = _qmul(_qmul(qa, j["rel_rotation"].astype(np.float64)), np.array([-qb[0], -qb[1], -qb[2], qb[3]]))
        ang = 2.0 * np.linalg.norm(d[:3])
    return np.linalg.norm(wa - wb), ang


def _integrate(xf, lin, ang, dt):
    for i in range(1, len(xf)):
        xf["position"][i] += (lin[i] * dt).astype(np.float32)
        q = xf["rotation"][i].astype(np.float64)
        q = q + 0.5 * dt * _qmul(np.append(ang[i], 0.0), q)
        xf["rotation"][i] = q / np.linalg.norm(q)


def test_an_initial_error_shrinks_for_every_type():
    """Two free bodies (and a body against the world) start with a position and an angular error; rows from joints_ref, solved by the row
    loop and integrated, must bring both down: this pins the sign of every bias."""
    dt = 1.0 / 60.0
    tilt = np.array([np.sin(0.2), 0.0, 0.0, np.cos(0.2)])   # 0.4 rad about x
    for type_ in range(4):
        for b in (0, 2):
            xf = np.zeros(3, scenes.TRANSFORM); xf["rotation"][:, 3] = 1.0
            xf["position"][1] = (0.3, 1.2, -0.2); xf["position"][2] = (0.0, 0.0, 0.1)
            xf["rotation"][1] = tilt; xf["rotation"][2] = (0.0, np.sin(-0.15), 0.0, np.cos(-0.15))
            j = _joint(type_, 1, b, anchor_a=(0.0, -0.5, 0.0), anchor_b=(0.0, 0.5, 0.0), length=0.25)
            joints = np.array([j])
            lin, ang = np.zeros((3, 3)), np.zeros((3, 3))
            minv, inv_i = np.array([0.0, 1.0, 0.5]), np.stack([np.zeros((3, 3)), np.eye(3) * 2.0, np.eye(3)])
            p0, a0 = _errors(joints[0], xf)
            assert p0 > 0.2 and (a0 > 0.2 or type_ in (joints_ref.BALL, joints_ref.DISTANCE))
            for step in range(120):
                rows = joints_ref.joint_rows(joints, xf, dt)
                rows_ref.apply_rows(rows, lin, ang, minv, inv_i, warm=True)
                for _ in range(8):
                    rows_ref.apply_rows(rows, lin, ang, minv, inv_i)
                joints_ref.set_impulses(joints, rows)
                _integrate(xf, lin, ang, dt)
            p1, a1 = _errors(joints[0], xf)
            assert p1 < 0.05 * p0, (type_, b, p0, p1)
            assert a1 < 0.05 * max(a0, 1e-9) or a0 == 0.0 or type_ in (joints_ref.BALL, joints_ref.DISTANCE), (type_, b, a0, a1)


def test_distance_rows_fall_back_when_the_anchors_coincide():
    xf = np.zeros(2, scenes.TRANSFORM); xf["rotation"][:, 3] = 1.0
    r = joints_ref.joint_rows([_joint(joints_ref.DISTANCE, 1, 0, length=0.5)], xf, 0.01)[0]
    assert tuple(r["lin_a"]) == (0.0, 1.0, 0.0) and r["bias"] == np.float32(np.float32(0.2) / np.float32(0.01)) * np.float32(-0.5)


def test_levels_follow_shared_bodies():
    ab = [(1, 0), (2, 1), (3, 0), (3, 2), (4, 0), (1, 4)]
    joints = np.array([_joint(i % 4, a, b) for i, (a, b) in enumerate(ab)])
    assert list(joints_ref.joint_levels(joints)) == [0, 1, 0, 2, 0, 2]
    assert list(joints_ref.table_order(joints)) == [0, 2, 4, 1, 3, 5]


def test_joint_layout_matches_the_header(tmp_path):
    fields = nudge_b200.JOINT.names
    src = tmp_path / "layout.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "nudge_b200.h"\nint main(void) {\n' +
                   "".join('printf("%%zu\\n", offsetof(nb_joint, %s));\n' % f for f in fields) +
                   'printf("%zu\\n", sizeof(nb_joint)); return 0; }\n')
    exe = tmp_path / "layout"
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), "-o", str(exe), str(src)])
    out = [int(x) for x in subprocess.check_output([str(exe)]).split()]
    assert out[:-1] == [abi.JOINT.fields[f][1] for f in fields]
    assert out[-1] == abi.JOINT.itemsize == 112
