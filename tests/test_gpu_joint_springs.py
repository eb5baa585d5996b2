"""Joint springs (nb_upload_joint_springs; DESIGN.md section 8.21): the spring table and the spring rows byte for byte against the numpy
restatement (tests/joint_spring_ref.py) with drives and broken joints mixed in; runs byte for byte against a twin fed the restated rows
through nb_upload_constraint_rows; slider, hinge and distance springs following the backward-Euler recurrence, a two-link arm holding its
targets under gravity and a powered ragdoll ball reaching its target, all under graph replays; targets uploaded every step keeping the
graph and the launches; snapshots with every table present, state files, body removal, joint uploads and the refusals."""
import numpy as np
import pytest
import nudge_b200
from nudge_b200 import scenes, abi
from oracle import joints_ref
from tests import joint_dof_ref as dof
from tests import joint_spring_ref as spr
from tests.gpu_util import side_stream, joint_rows
from tests.test_gpu_rows import _free_bodies, _pile, _quat_rotate
from tests.test_gpu_joints import _joints_at_rest, _body_bytes
from tests.test_gpu_joint_drives import _renumber
from tests.test_gpu_joint_dof import _random_drives, _dof_drives_on_all, _coordinates, _link
from tests.test_joint_springs_ref import spring, _recurrence
from tests.test_joint_spring_geometry_ref import cases as geometry_cases, check_spring
from tests.test_gpu_joint_geometry import _scene as _geometry_scene

pytestmark = pytest.mark.gpu
ROWS = joints_ref.ROWS_PER_TYPE
BALL, HINGE, FIXED, DISTANCE = joints_ref.BALL, joints_ref.HINGE, joints_ref.FIXED, joints_ref.DISTANCE


def _random_springs(joints, rng, share=0.6):
    out = []
    for i, j in enumerate(joints):
        if rng.random() > share:
            continue
        t = int(j["type"])
        s = np.zeros(1, nudge_b200.JOINT_SPRING)[0]
        s["joint"] = i
        if t == BALL:
            s["target"] = scenes._random_unit_quaternions(rng, 1)[0]
        else:
            s["target"][0] = rng.uniform(-np.pi, np.pi) if t == HINGE else rng.uniform(-1.0, 1.0) if t == FIXED else rng.uniform(0.0, 3.0)
            s["target_velocity"] = rng.normal() * 0.5
        s["stiffness"] = rng.uniform(0.0, 100.0) if rng.random() < 0.9 else 0.0
        s["damping"] = rng.uniform(0.1, 5.0) if rng.random() < 0.8 or s["stiffness"] == 0 else 0.0
        s["max_force"] = np.inf if rng.random() < 0.5 else rng.uniform(0.0, 20.0)
        s["impulse"] = rng.normal(size=3) * 0.01 * np.array([1.0, t == BALL, t == BALL])
        out.append(s)
    return np.array(out, nudge_b200.JOINT_SPRING)


def test_own_rows_drive_rows_and_table_equal_the_numpy_restatement_byte_for_byte():
    n, m = 60, 320
    s, rng = _free_bodies(n, 4)
    g = nudge_b200.Sim(s)
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
    drives = _random_drives(joints, rng, share=0.5, broken=0.05, fragile=0.1)
    springs = _random_springs(joints, rng)
    assert {int(joints[int(x)]["type"]) for x in springs["joint"]} == {BALL, HINGE, FIXED, DISTANCE}
    g.upload_joints(joints); g.upload_joint_drives(drives); g.upload_joint_springs(springs)
    order = joints_ref.table_order(joints)
    jt = joints[order]
    want_stable, want_simp = spr.spring_table(jt, _renumber(springs, order))
    stable = g.debug("joint_springs", spr.SPRING_TABLE)
    assert stable.tobytes() == want_stable.tobytes()
    assert g.debug("joint_spring_rows", nudge_b200.ROW)["impulse"].tobytes() == want_simp.tobytes()
    table = g.debug("joint_drives", dof.DRIVE_TABLE)
    before = joint_rows(g)
    n_own = int(sum(ROWS[t] for t in joints["type"]))
    g.collide(); g.apply_gravity_damping(); g.read_cached_impulses(); g.setup_contact_constraints()
    got, sgot = joint_rows(g), g.debug("joint_spring_rows", nudge_b200.ROW)
    g.download_bodies()
    dt = np.float32(s.time_step)
    table["broken"] = dof.broken_after(jt, before, table, dt)
    sprung = stable["present"] != 0
    assert 0 < table["broken"][sprung].sum() < sprung.sum()
    want, swant = spr.joint_rows(jt, g.transforms, dt, table, before["impulse"][n_own:], stable, want_simp)
    assert len(sgot) == len(swant) == sum(spr.spring_row_count(int(joints[int(x)]["type"])) for x in springs["joint"])
    for k in nudge_b200.ROW.names:
        assert got[k].tobytes() == want[k].tobytes(), k
        assert sgot[k].tobytes() == swant[k].tobytes(), k
    assert g.debug("joint_springs", spr.SPRING_TABLE).tobytes() == stable.tobytes()
    g.apply_impulses(int(s.iterations)); g.update_cached_impulses(); g.write_cached_impulses(); g.advance()
    back = g.download_joint_springs()
    ss = np.sort(springs, order="joint")
    assert list(back["joint"]) == list(ss["joint"])
    for k in ("target", "target_velocity", "stiffness", "damping", "max_force"):
        assert back[k].tobytes() == ss[k].tobytes(), k
    pos = stable[np.argsort(order)][back["joint"]]
    broken = table[np.argsort(order)][back["joint"]]["broken"]
    for p, sp, e, br in zip(back["position"], back, pos, broken):
        if not br:
            assert np.float32(p).tobytes() == np.float32(spr.spring_position(int(joints[int(sp["joint"])]["type"]), e["position"])).tobytes()


def test_device_spring_rows_against_the_float64_geometry():
    """Every spring row of tests/test_joint_spring_geometry_ref.cases() built by the device, each joint's pair in a cell of its own, checked
    by check_spring: Jacobian, C, softness, bounds and the downloaded position against float64 geometry."""
    cases = geometry_cases()
    m = len(cases)
    s = _geometry_scene(2 * m)
    joints = np.zeros(m, nudge_b200.JOINT)
    springs = []
    grid = int(np.ceil(m ** (1.0 / 3.0)))
    for k, (j, sp, xf, _) in enumerate(cases):
        a, b = 2 * k + 1, 2 * k + 2
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
        sp = sp.copy(); sp["joint"] = k
        springs.append(sp)
    springs = np.array(springs, nudge_b200.JOINT_SPRING)
    g = nudge_b200.Sim(s)
    g.upload_joints(joints); g.upload_joint_springs(springs)
    g.collide(); g.apply_gravity_damping(); g.read_cached_impulses(); g.setup_contact_constraints()
    srows = g.debug("joint_spring_rows", nudge_b200.ROW)
    table = g.debug("joint_springs", spr.SPRING_TABLE)
    g.download_bodies()
    back = g.download_joint_springs()
    rng = np.random.default_rng(5)
    for p, i in enumerate(joints_ref.table_order(joints)):
        e = table[p]
        rows = srows[e["row"]:e["row"] + spr.spring_row_count(int(joints[i]["type"]))]
        check_spring(joints[i], springs[i], g.transforms, rows, e, rng, off=cases[i][3], dt=np.float32(s.time_step), where="joint %d" % i)
        assert np.float32(back["position"][i]).tobytes() == np.float32(spr.spring_position(int(joints[i]["type"]), e["position"])).tobytes()


def test_a_new_target_wakes_a_sleeping_body():
    """A slider spring at rest on its target: after 255 slow steps the body sleeps, and an upload with a new target wakes it and moves it."""
    s, joints, drives = _rig()
    _unit_bodies(s, [1])
    g = nudge_b200.Sim(s, stream=side_stream())
    g.upload_joints(joints[:1]); g.upload_joint_drives(drives)
    g.upload_joint_springs(np.array([spring(0, 0.0, 30.0, 10.0)]))
    for _ in range(300):
        g.step()
    g.download_bodies()
    assert g.idle[1] == 255
    before = _coordinates(joints[0], g.transforms)[3]
    g.upload_joint_springs(np.array([spring(0, 0.5, 30.0, 10.0)]))
    g.download_bodies()
    assert g.idle[1] == 0
    for _ in range(240):
        g.step()
    g.download_bodies()
    assert abs(before) < 1e-3 and abs(_coordinates(joints[0], g.transforms)[3] - 0.5) < 0.01


def _twin_run(s, mode, steps, settle, m, seed):
    """x runs with joints, drives and springs; y gets the restated rows in solve order through nb_upload_constraint_rows."""
    rng = np.random.default_rng(seed)
    x, y = nudge_b200.Sim(s), nudge_b200.Sim(s)
    for g in (x, y):
        g.set_solver_mode(mode)
        for _ in range(settle):
            g.step_staged()
    y.download_bodies()
    joints = _joints_at_rest(y.transforms, rng, m, s.n_bodies)
    drives = _dof_drives_on_all(joints, rng)
    springs = _random_springs(joints, rng, share=0.7)
    springs["max_force"] = np.where(np.isinf(springs["max_force"]), np.inf, springs["max_force"] + 1.0)
    x.upload_joints(joints); x.upload_joint_drives(drives); x.upload_joint_springs(springs)
    yj = joints.copy()
    table, imp = dof.drive_table(yj, drives)
    stable, simp = spr.spring_table(yj, springs)
    order = spr.solve_order(yj, table, stable)
    n_own = int(sum(ROWS[t] for t in joints["type"]))
    dt = np.float32(s.time_step)
    for step in range(steps):
        y.download_bodies()
        rows, srows = spr.joint_rows(yj, y.transforms, dt, table, imp, stable, simp)
        allr = np.concatenate([rows, srows])
        y.upload_constraint_rows(allr[order])
        x.step_staged(); y.step_staged()
        allr[order] = y.download_constraint_rows(len(allr))
        joints_ref.set_impulses(yj, allr[:n_own]); imp = allr["impulse"][n_own:len(rows)].copy(); simp = allr["impulse"][len(rows):].copy()
        x.download_bodies(); y.download_bodies()
        assert x.momentum.tobytes() == y.momentum.tobytes(), step
        assert x.transforms.tobytes() == y.transforms.tobytes(), step
        assert x.download_joints()["impulse"].tobytes() == yj["impulse"].tobytes(), step
        xs = x.download_joint_springs()
        want = np.zeros((len(xs), 3), np.float32)
        for r, sp in enumerate(xs):
            e = stable[int(sp["joint"])]
            c = spr.spring_row_count(int(yj[int(sp["joint"])]["type"]))
            want[r, :c] = simp[e["row"]:e["row"] + c]
        assert xs["impulse"].tobytes() == want.tobytes(), step
    assert np.isfinite(x.transforms["position"]).all()


def test_springs_equal_the_row_path_among_contacts_in_parity_mode():
    _twin_run(_pile(), "parity", 60, 30, 48, 13)


def test_springs_equal_the_row_path_in_throughput_mode_without_contacts():
    s, _ = _free_bodies(40, 5)
    _twin_run(s, "throughput", 60, 0, 36, 5)


def _unit_bodies(s, bodies):
    """Mass 1 and inertia I / 12 for `bodies`, boxes too small to touch each other (box k is body k's), and rest."""
    s.properties["mass_inverse"][bodies] = 1.0; s.properties["inertia_inverse"][bodies] = 12.0
    s.box_data["size"][bodies] = 0.05
    s.transforms["rotation"][:] = (0.0, 0.0, 0.0, 1.0)
    s.momentum["velocity"][:] = 0.0; s.momentum["angular_velocity"][:] = 0.0


def _rig():
    """Three free bodies far apart without gravity or damping: body 1 on a slider along x, body 2 on a hinge about y, body 3 on a distance
    joint, each to the world with its anchor at the body's centre (on the axis)."""
    s, _ = _free_bodies(3, 8)
    xf = s.transforms
    xf["rotation"][:] = (0.0, 0.0, 0.0, 1.0)
    s.momentum["velocity"][:] = 0.0; s.momentum["angular_velocity"][:] = 0.0
    for k in (1, 2, 3):
        xf["position"][k] = (100.0 * k, 500.0, 0.0)
    joints = [_link(FIXED, 1, 0, xf["position"][1], xf, (1, 0, 0)), _link(HINGE, 2, 0, xf["position"][2], xf, (0, 1, 0))]
    rope = _link(DISTANCE, 3, 0, xf["position"][3] + np.float32([0.0, 1.5, 0.0]), xf, (0, 1, 0))
    rope["anchor_a"] = 0.0; rope["length"] = 1.5
    joints.append(rope)
    d = np.zeros(1, nudge_b200.JOINT_DRIVE); d["joint"], d["flags"], d["break_force"], d["break_torque"] = 0, dof.SLIDE, np.inf, np.inf
    return s, np.array(joints), d


def test_slider_hinge_and_distance_springs_follow_the_recurrence_over_graph_replays():
    s, joints, drives = _rig()
    g = nudge_b200.Sim(s, stream=side_stream())
    g.upload_joints(joints); g.upload_joint_drives(drives)
    mass = 1.0 / s.properties["mass_inverse"][1:4].astype(np.float64)
    inertia_y = 1.0 / float(s.properties["inertia_inverse"][2][1])
    cases = [(0, 0.3, 30.0, 0.5, mass[0]), (1, 0.05, 2.0 * inertia_y * 60, 0.0, inertia_y), (2, 1.2, 40.0, 1.0, mass[2])]
    springs = np.array([spring(j, t, k, c) for j, t, k, c, _ in cases])
    g.upload_joint_springs(springs)
    got = []
    for _ in range(300):
        g.step()
        g.download_bodies()
        _, _, angle, s_, _ = zip(*[_coordinates(j, g.transforms) for j in joints[:2]])
        dist = np.linalg.norm(g.transforms["position"][3].astype(np.float64) - (joints[2]["anchor_b"]).astype(np.float64))
        got.append((s_[0], angle[1], dist))
    assert g.debug_scalar("graph_records") == 1
    got = np.array(got)
    x0 = (0.0, 0.0, 1.5)
    for i, (j, t, k, c, m) in enumerate(cases):
        want = _recurrence(x0[i], t, k, c, m, 300, dt=float(s.time_step))
        amp = abs(x0[i] - t)
        tol = 3e-3 * amp if i == 1 else 1e-3 * amp
        assert np.abs(got[:, i] - want).max() < tol, (i, np.abs(got[:, i] - want).max(), tol)
    back = g.download_joint_springs()
    assert abs(back["position"][0] - got[-2, 0]) < 1e-4 and abs(back["position"][2] - got[-2, 2]) < 1e-4


def test_two_link_arm_holds_its_targets_under_gravity():
    """A shoulder hinge to the world and an elbow hinge, both about z, the links horizontal at rest: steady-state error load / k within 2 %."""
    s, _ = _free_bodies(2, 16)
    s.gravity = np.float32(9.82)
    _unit_bodies(s, [1, 2])
    xf = s.transforms
    o = np.array([0.0, 500.0, 0.0], np.float32)
    xf["position"][1] = o + np.float32([0.5, 0.0, 0.0]); xf["position"][2] = o + np.float32([1.5, 0.0, 0.0])
    joints = np.array([_link(HINGE, 1, 0, o, xf, (0, 0, 1)), _link(HINGE, 2, 1, o + np.float32([1.0, 0.0, 0.0]), xf, (0, 0, 1))])
    m = (1.0, 1.0)
    # about 0.05 rad of sag at each joint; damping ratios near 0.5 on the inertia each joint moves (2.7 and 0.33 about z), so that the arm
    # settles well before its bodies are slow enough for long enough to fall asleep
    k = (400.0, 100.0)
    springs = np.array([spring(0, 0.0, k[0], np.sqrt(k[0] * 2.7)), spring(1, 0.0, k[1], np.sqrt(k[1] * 0.33))])
    g = nudge_b200.Sim(s, stream=side_stream())
    g.upload_joints(joints); g.upload_joint_springs(springs)
    for i in range(1200):
        if i % 200 == 0:   # keep the slowly settling arm awake (a body slow for 255 steps sleeps): its own velocities, idle counter 0
            g.set_body_states(g.get_body_states([1, 2]), abi.BODY_VELOCITY)
        g.step()
    g.download_bodies()
    assert (g.idle[1:3] < 255).all()
    p = g.transforms["position"].astype(np.float64)
    # gravity's torque about z at each joint on what lies beyond it; the arm sags by about load / k
    elbow = _quat_rotate(g.transforms["rotation"][1].astype(np.float64), joints[1]["anchor_b"].astype(np.float64)) + p[1]
    load = (-9.82 * (m[0] * (p[1][0] - o[0]) + m[1] * (p[2][0] - o[0])), -9.82 * m[1] * (p[2][0] - elbow[0]))
    theta = [_coordinates(j, g.transforms)[2] for j in joints]   # b relative to a: the shoulder's minus a's angle
    back = g.download_joint_springs()
    for i in range(2):
        sag = load[i] / k[i]
        assert abs(sag) > 0.01
        assert abs(abs(theta[i]) - abs(sag)) < 0.02 * abs(sag), (i, theta[i], sag)
        assert abs(back["position"][i] - theta[i]) < 1e-4


def test_powered_ragdoll_ball_reaches_its_target():
    s, _ = _free_bodies(2, 8)
    s.gravity = np.float32(9.82)
    _unit_bodies(s, [1, 2])
    xf = s.transforms
    o = np.array([0.0, 500.0, 0.0], np.float32)
    xf["position"][1] = o; xf["position"][2] = o + np.float32([0.0, -0.6, 0.0])
    joints = np.array([_link(FIXED, 1, 0, o, xf, (0, 1, 0)), _link(BALL, 2, 1, o + np.float32([0.0, -0.3, 0.0]), xf, (0, 1, 0))])
    axis = np.array([1.0, 0.0, 0.5]) / np.linalg.norm([1.0, 0.0, 0.5])
    target = np.append(np.sin(0.35) * axis, np.cos(0.35)).astype(np.float32)   # 0.7 rad
    g = nudge_b200.Sim(s, stream=side_stream())
    g.upload_joints(joints); g.upload_joint_springs(np.array([spring(1, target, 400.0, 20.0)]))
    for _ in range(300):
        g.step()
    g.download_bodies()
    q1, q2 = (g.transforms["rotation"][k].astype(np.float64) for k in (1, 2))
    rel = _qmul64(_conj64(q2), q1)   # conj(q_a) * q_b, a = body 2
    d = _qmul64(rel, _conj64(target.astype(np.float64)))
    err = 2.0 * np.arctan2(np.linalg.norm(d[:3]), abs(d[3]))
    assert err < 0.03, err   # gravity on the lower body's centre, 0.3 below the ball, holds it off by about load / k = 0.005
    back = g.download_joint_springs()
    assert abs(back["position"][0] - err) < 1e-3 and g.debug_scalar("graph_records") == 1


def _conj64(q):
    return np.array([-q[0], -q[1], -q[2], q[3]])


def _qmul64(l, r):
    return np.append(l[3] * r[:3] + r[3] * l[:3] + np.cross(l[:3], r[:3]), l[3] * r[3] - l[:3] @ r[:3])


def _pile_with_springs(seed, m=40, stream=True):
    s = _pile()
    g = nudge_b200.Sim(s, stream=side_stream()) if stream else nudge_b200.Sim(s)
    rng = np.random.default_rng(seed)
    joints = _joints_at_rest(s.transforms, rng, m, s.n_bodies)
    drives = _dof_drives_on_all(joints, rng)
    springs = _random_springs(joints, rng, share=0.8)
    g.upload_joints(joints); g.upload_joint_drives(drives); g.upload_joint_springs(springs)
    return s, g, joints, drives, springs, rng


def test_targets_uploaded_every_step_keep_the_graph_add_no_launch_and_leave_the_drive_rows():
    s, g, joints, drives, springs, rng = _pile_with_springs(8)
    base = nudge_b200.Sim(s, stream=side_stream())
    base.upload_joints(joints); base.upload_joint_drives(drives)
    base.step()
    before = base.launch_count(); base.step(); without = base.launch_count() - before
    per_step = []
    for step in range(100):
        for sp in springs:
            t = int(joints[int(sp["joint"])]["type"])
            if t != BALL:
                sp["target"][0] = rng.uniform(-1.0, 1.0) if t != DISTANCE else rng.uniform(0.5, 2.0)
        springs["stiffness"] = rng.uniform(1.0, 50.0, len(springs))
        g.upload_joint_springs(springs)
        before = g.launch_count(); g.step(); per_step.append(g.launch_count() - before)
    assert g.debug_scalar("graph_records") == 1 and set(per_step) == {without}
    g.upload_joint_springs(springs[1:])   # another structure: one new record
    for _ in range(3):
        g.step()
    assert g.debug_scalar("graph_records") == 2
    g.upload_joint_springs(None)
    assert len(g.debug("joint_spring_rows", nudge_b200.ROW)) == 0 and len(g.download_joint_springs()) == 0
    before = g.launch_count(); g.step()
    assert g.launch_count() - before == without
    g.download_bodies()
    assert len(joint_rows(g)) == sum(ROWS[t] for t in joints["type"]) + sum(dof.drive_row_count(int(f)) for f in drives["flags"])


def test_snapshot_restore_repeats_a_run_with_every_table_present():
    from tests.test_gpu_snapshot import _scene, _sim
    s, rows = _scene()
    x = _sim(s, rows)
    x.enable_contact_events(1 << 16)
    rng = np.random.default_rng(3)
    x.step()
    x.download_bodies()
    joints = _joints_at_rest(x.transforms, rng, 20, s.n_bodies)
    x.upload_joints(joints); x.upload_joint_drives(_dof_drives_on_all(joints, rng)); x.upload_joint_springs(_random_springs(joints, rng, share=1.0))
    x.upload_ccd_bodies([(b, 0.2, 0.1, 0xffff, 0xffff) for b in (300, 301, 302)])
    for _ in range(3):
        x.step()
    snap = x.snapshot()

    def run():
        for _ in range(20):
            x.step()
        return _body_bytes(x) + x.download_joints().tobytes() + x.download_joint_drives().tobytes() + x.download_joint_springs().tobytes()
    first = run()
    x.restore(snap)
    assert run() == first


def test_state_file_version_9_round_trip_and_a_version_8_file(tmp_path):
    s, g, joints, drives, springs, rng = _pile_with_springs(7, stream=False)
    h = nudge_b200.Sim(s)
    for _ in range(5):
        g.step()
    path = str(tmp_path / "springs.nbstate")
    g.save_state(path)
    raw = open(path, "rb").read()
    assert int.from_bytes(raw[8:12], "little") == 9
    h.load_state(path)
    a, b = g.download_joint_springs(), h.download_joint_springs()
    assert len(a) == len(springs) and a["impulse"].tobytes() == b["impulse"].tobytes() and a["target"].tobytes() == b["target"].tobytes()
    for _ in range(5):
        g.step(); h.step()
    assert _body_bytes(g) == _body_bytes(h) and h.download_joint_springs().tobytes() == g.download_joint_springs().tobytes()
    # a context with a continuous-collision set and no springs writes version 8; loading it removes the springs
    k = nudge_b200.Sim(s)
    k.upload_joints(joints); k.upload_ccd_bodies([(5, 0.2, 0.1, 0xffff, 0xffff)])
    old = str(tmp_path / "v8.nbstate")
    k.save_state(old)
    assert int.from_bytes(open(old, "rb").read()[8:12], "little") == 8
    g.load_state(old)
    assert len(g.download_joint_springs()) == 0 and len(g.debug("joint_springs", spr.SPRING_TABLE)) == 0
    # without springs nothing changes in the file
    k.upload_joint_springs(springs[:3]); k.upload_joint_springs(None)
    again = str(tmp_path / "v8b.nbstate")
    k.save_state(again)
    assert open(again, "rb").read() == open(old, "rb").read()


def test_body_removal_renumbers_springs_and_joint_uploads_keep_or_drop_them():
    s, g, joints, drives, springs, rng = _pile_with_springs(4, m=60, stream=False)
    for _ in range(3):
        g.step()
    before_j, before_s = g.download_joints(), g.download_joint_springs()
    gone = np.array([int(joints[5]["a"]), 57, 130], np.uint32)
    g.remove_bodies(gone)
    keep = ~(np.isin(before_j["a"], gone) | np.isin(before_j["b"], gone))
    new_index = np.cumsum(keep) - 1
    want = before_s[keep[before_s["joint"]]].copy()
    want["joint"] = new_index[want["joint"]]
    got = g.download_joint_springs()
    assert 0 < len(got) < len(before_s)
    for k in ("joint", "target", "target_velocity", "stiffness", "damping", "max_force", "impulse"):
        assert got[k].tobytes() == want[k].tobytes(), k
    for _ in range(3):
        g.step()
    j2 = g.download_joints()
    g.upload_joints(j2)   # the same structure: the springs stay
    assert len(g.download_joint_springs()) == len(got)
    g.upload_joints(j2[1:])   # another structure: they go
    assert len(g.download_joint_springs()) == 0
    g.download_bodies()
    assert np.isfinite(g.transforms["position"]).all()


def test_refusals_change_nothing():
    s, g, joints, drives, springs, rng = _pile_with_springs(9, m=20, stream=False)
    kept = g.download_joint_springs().tobytes()
    types = joints["type"]
    ball, fixed, hinge = (int(np.flatnonzero(types == t)[0]) for t in (BALL, FIXED, HINGE))
    dist = int(np.flatnonzero(types == DISTANCE)[0])
    unit = (0.0, 0.0, 0.0, 1.0)

    def one(joint, target, k=1.0, **kw):
        d = np.array([spring(joint, target, k)])
        for key, v in kw.items():
            d[0][key] = v
        return d
    cases = [(one(len(joints), 0.0), "at or beyond the joint count"), (np.concatenate([one(hinge, 0.0), one(hinge, 0.1)]), "two springs on joint"),
             (one(hinge, 0.0, reserved=1), "reserved"), (one(hinge, np.nan), "not finite"), (one(hinge, 0.0, damping=np.inf), "not finite"),
             (one(hinge, 0.0, max_force=np.nan), "max_force"), (one(hinge, 0.0, max_force=-np.inf), "max_force"),
             (one(hinge, 0.0, k=-1.0), "negative"), (one(hinge, 0.0, damping=-1.0), "negative"), (one(hinge, 0.0, max_force=-1.0), "negative"),
             (one(hinge, 0.0, k=0.0), "both 0"), (one(hinge, (0.0, 1.0)), "does not read"), (one(fixed, (0.0, 0.0, 0.0, 1.0)), "does not read"),
             (one(hinge, 3.2), r"outside \[-pi, pi\]"), (one(dist, -0.1), "negative distance"), (one(ball, unit, target_velocity=1.0), "target velocity"),
             (one(ball, (0.0, 0.0, 0.0, 1.01)), "not of unit length"), (one(hinge, 0.0, k=1e-37), r"outside \{0\} and \[1e-12, 1e12\]"),
             (one(hinge, 0.0, k=2e12), "outside"), (one(hinge, 0.0, damping=1e-20), "outside"), (one(hinge, 0.0, target_velocity=2e12), "target velocity beyond"),
             (one(fixed, 3e12), "target beyond"), (one(dist, 3e12), "target beyond")]
    for d, what in cases:
        with pytest.raises(nudge_b200.NudgeError, match=what):
            g.upload_joint_springs(d)
        assert g.download_joint_springs().tobytes() == kept
    with pytest.raises(nudge_b200.NudgeError, match="null spring list"):
        g._ck(g.lib.nb_upload_joint_springs(g.ctx, None, 1, g.stream), "nb_upload_joint_springs")
    bent = joints.copy(); bent[fixed]["axis_a"] = (0.0, 0.0, 0.9); bent[hinge]["rel_rotation"] = (0.0, 0.0, 0.0, 1.01)
    g.upload_joints(bent)   # the same structure: the springs stay
    for d, what in ((one(fixed, 0.0), "axis_a is not of unit length"), (one(hinge, 0.0), "rel_rotation is not of unit length")):
        with pytest.raises(nudge_b200.NudgeError, match=what):
            g.upload_joint_springs(d)
    assert g.download_joint_springs().tobytes() == kept
    g.upload_joints(joints)
    import ctypes as C
    n = C.c_uint32(0)
    assert g.lib.nb_download_joint_springs(g.ctx, None, 0, C.byref(n), g.stream) == -2 and n.value == len(springs)   # NB_ERR_CAPACITY
    g.upload_joint_springs(one(hinge, np.float32(np.pi), max_force=np.inf))
    assert len(g.download_joint_springs()) == 1
