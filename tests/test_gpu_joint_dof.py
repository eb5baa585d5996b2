"""Sliders and swing-twist limits (NB_JOINT_SLIDE, NB_JOINT_CONE, NB_JOINT_TWIST; DESIGN.md section 8.20): the drive table and every row byte
for byte against the numpy restatement (tests/joint_dof_ref.py) with old and new flags mixed; runs byte for byte against a twin fed the
restated rows through nb_upload_constraint_rows, breaks included; a ragdoll, a motorised piston and a sliding door under one graph record;
the graph and launch rules; snapshots, state files and body removal; and the new refusals."""
import numpy as np
import pytest
import nudge_b200
from nudge_b200 import scenes
from oracle import joints_ref
from tests import joint_dof_ref as dof
from tests.gpu_util import side_stream, joint_rows
from tests.test_gpu_rows import _free_bodies, _pile, _quat_rotate
from tests.test_gpu_joints import _joints_at_rest, _body_bytes
from tests.test_gpu_joint_drives import _renumber, _breaks_mid_run, _without_position

pytestmark = pytest.mark.gpu
ROWS = joints_ref.ROWS_PER_TYPE
BALL, HINGE, FIXED, DISTANCE = joints_ref.BALL, joints_ref.HINGE, joints_ref.FIXED, joints_ref.DISTANCE
L, M, BR, S, CN, TW = dof.LIMIT, dof.MOTOR, dof.BREAKABLE, dof.SLIDE, dof.CONE, dof.TWIST


def _flags(t, rng):
    """Random flags joint type t takes, new and old mixed."""
    r = int(rng.integers(0, 8))
    if t == BALL:
        return (CN if r & 1 else 0) | (TW if r & 2 else 0) | (BR if r & 4 else 0)
    if t == FIXED:
        return S | (r & (L | M | BR)) if rng.random() < 0.7 else r & BR
    return r & (L | M | BR if t == HINGE else L | BR)


def _random_drives(joints, rng, share=0.8, broken=0.0, fragile=0.0):
    out = []
    for i, j in enumerate(joints):
        if rng.random() > share:
            continue
        t = int(j["type"])
        d = np.zeros(1, nudge_b200.JOINT_DRIVE)[0]
        d["joint"], d["flags"] = i, _flags(t, rng)
        if t in (HINGE, BALL):
            d["lower"], d["upper"] = np.sort(rng.uniform(-np.pi, np.pi, 2))
        else:
            d["lower"], d["upper"] = np.sort(rng.uniform(0.0, 3.0, 2)) - (1.5 if t == FIXED else 0.0)
        if d["flags"] & CN:
            d["cone"] = rng.uniform(0.05, np.pi)
        else:
            d["motor_speed"], d["max_motor_torque"] = rng.normal() * 2.0, rng.random() * 5.0
        d["break_force"], d["break_torque"] = (0.0, 0.0) if rng.random() < fragile else (np.inf, rng.random() * 50.0 if rng.random() < 0.5 else np.inf)
        d["impulse"] = rng.normal(size=3) * 0.01
        d["broken"] = 1 if rng.random() < broken else 0
        out.append(d)
    return np.array(out, nudge_b200.JOINT_DRIVE)


def _drive_impulses(joints, table, imp, driven):
    """The impulse[3] (motor or cone, lower, upper) of the drives on the joints `driven`, from the appended rows' impulses in joint order."""
    out, m = {}, 0
    for i in range(len(joints)):
        fl = int(table["flags"][i])
        v = np.zeros(3, np.float32)
        for k in range(3):
            if fl & (dof.RANGE if k else dof.FIRST):
                v[k] = imp[m]; m += 1
        out[i] = v
    return np.array([out[i] for i in driven], np.float32).reshape(-1, 3)


def test_own_rows_drive_rows_and_table_equal_the_numpy_restatement_byte_for_byte():
    n = 60
    s, rng = _free_bodies(n, 4)
    g = nudge_b200.Sim(s)
    m = 400
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
    drives = _random_drives(joints, rng, broken=0.05, fragile=0.1)
    flags = set(int(f) for f in drives["flags"])
    assert {S, S | L | M | BR, CN, TW, CN | TW | BR, L | M} <= flags
    g.upload_joints(joints); g.upload_joint_drives(drives)
    order = joints_ref.table_order(joints)
    table = g.debug("joint_drives", dof.DRIVE_TABLE)
    before = joint_rows(g)
    n_own = int(sum(ROWS[t] for t in joints["type"]))
    want_table, want_imp = dof.drive_table(joints[order], _renumber(drives, order))
    assert table.tobytes() == want_table.tobytes()
    assert before["impulse"][n_own:].tobytes() == want_imp.tobytes()
    g.collide(); g.apply_gravity_damping(); g.read_cached_impulses(); g.setup_contact_constraints()
    got = joint_rows(g)
    g.download_bodies()
    dt = np.float32(s.time_step)
    jt = joints[order]
    table["broken"] = dof.broken_after(jt, before, table, dt)
    new = (table["flags"] & (S | CN | TW)) != 0
    assert 0 < table["broken"][new].sum() < new.sum() and table["broken"].sum() > drives["broken"].sum()
    want = dof.joint_rows(jt, g.transforms, dt, table, before["impulse"][n_own:])
    assert len(got) == len(want) == n_own + sum(dof.drive_row_count(int(f)) for f in drives["flags"])
    for k in nudge_b200.ROW.names:
        assert got[k].tobytes() == want[k].tobytes(), k
    assert g.debug("joint_drives", dof.DRIVE_TABLE).tobytes() == table.tobytes()
    g.apply_impulses(int(s.iterations)); g.update_cached_impulses(); g.write_cached_impulses(); g.advance()
    back = g.download_joint_drives()
    sd = np.sort(drives, order="joint")
    assert list(back["joint"]) == list(sd["joint"])
    cone = (sd["flags"] & CN) != 0
    for k in ("flags", "lower", "upper", "break_force", "break_torque"):
        assert back[k].tobytes() == sd[k].tobytes(), k
    assert back["cone"].tobytes() == np.where(cone, sd["cone"], 0).astype(np.float32).tobytes()
    for k in ("motor_speed", "max_motor_torque"):
        assert back[k].tobytes() == np.where(cone, 0, sd[k]).astype(np.float32).tobytes(), k
    pos = table[np.argsort(order)][back["joint"]]
    want_pos = [dof.drive_position(int(joints[j]["type"]), int(e["flags"]), e["position"]) if not e["broken"] else None for j, e in zip(back["joint"], pos)]
    for p, w, e in zip(back["position"], want_pos, pos):
        if w is not None:
            assert np.float32(p).tobytes() == np.float32(w).tobytes(), e


def _twin_run(s, joints_of, drives_of, mode, steps, settle, edit_at):
    """x runs with joints and drives; y gets the restated rows (joint order: own rows, then the drive's) through nb_upload_constraint_rows,
    with the break rule applied from its downloaded impulses.  At edit_at[0] a new drive list edit_at[1](download) goes to both."""
    x, y = nudge_b200.Sim(s), nudge_b200.Sim(s)
    for g in (x, y):
        g.set_solver_mode(mode)
        for _ in range(settle):
            g.step_staged()
    y.download_bodies()
    joints = joints_of(y.transforms)
    drives = drives_of(joints)
    x.upload_joints(joints); x.upload_joint_drives(drives)
    yj = joints.copy()
    table, imp = dof.drive_table(yj, drives)
    order = dof.solve_order(yj, table)
    n_own = int(sum(ROWS[t] for t in joints["type"]))
    dt = np.float32(s.time_step)
    prev, broke_at = None, None
    for step in range(steps):
        if step == edit_at[0]:
            drives = edit_at[1](x.download_joint_drives())
            x.upload_joint_drives(drives)
            table, imp = dof.drive_table(yj, drives)
            order = dof.solve_order(yj, table)
        if prev is not None:
            table["broken"] = dof.broken_after(yj, prev, table, dt)
        y.download_bodies()
        rows = dof.joint_rows(yj, y.transforms, dt, table, imp)
        y.upload_constraint_rows(rows[order])
        x.step_staged(); y.step_staged()
        rows[order] = y.download_constraint_rows(len(rows))
        joints_ref.set_impulses(yj, rows[:n_own]); imp = rows["impulse"][n_own:].copy()
        prev = rows
        xd = x.download_joint_drives()
        x.download_bodies(); y.download_bodies()
        assert x.momentum.tobytes() == y.momentum.tobytes(), step
        assert x.transforms.tobytes() == y.transforms.tobytes(), step
        assert x.download_joints()["impulse"].tobytes() == yj["impulse"].tobytes(), step
        assert xd["impulse"].tobytes() == _drive_impulses(yj, table, imp, xd["joint"]).tobytes(), step
        assert xd["broken"].tobytes() == table["broken"][xd["joint"]].tobytes(), step
        if broke_at is None and xd["broken"].any():
            broke_at = step
    assert np.isfinite(x.transforms["position"]).all()
    return broke_at


def _dof_drives_on_all(joints, rng):
    """A drive on every joint, BREAKABLE with infinite thresholds; every ball a CONE | TWIST, every weld a slider with LIMIT and MOTOR."""
    d = _random_drives(joints, rng, share=1.0)
    d["break_force"] = np.inf; d["break_torque"] = np.inf; d["broken"] = 0
    for e in d:
        t = int(joints[int(e["joint"])]["type"])
        if t == BALL:
            e["flags"], e["cone"], e["motor_speed"], e["max_motor_torque"] = CN | TW | BR, rng.uniform(0.3, 1.5), 0.0, 0.0
            e["lower"], e["upper"] = -rng.uniform(0.2, 1.0), rng.uniform(0.2, 1.0)
        elif t == FIXED:
            e["flags"], e["lower"], e["upper"] = S | L | M | BR, -rng.uniform(0.1, 0.5), rng.uniform(0.1, 0.5)
        else:
            e["flags"] = int(e["flags"]) | BR
    return d


def _first_new(joints, drives):
    return int(next(int(e["joint"]) for e in drives if int(e["flags"]) & (S | CN)))


def test_dof_drives_equal_the_row_path_among_contacts_in_parity_mode():
    s = _pile()
    rng = np.random.default_rng(13)
    held = {}

    def drives_of(j):
        held["d"] = _dof_drives_on_all(j, rng)
        return held["d"]
    broke_at = _twin_run(s, lambda xf: _joints_at_rest(xf, rng, 48, s.n_bodies), drives_of, "parity", 60, 30,
                         edit_at=(25, lambda d: _breaks_mid_run(None, _first_new(None, held["d"]))(d)))
    assert broke_at == 25


def test_dof_drives_equal_the_row_path_in_throughput_mode_without_contacts():
    s, rng = _free_bodies(40, 5)
    held = {}

    def drives_of(j):
        held["d"] = _dof_drives_on_all(j, rng)
        return held["d"]
    broke_at = _twin_run(s, lambda xf: _joints_at_rest(xf, rng, 36, s.n_bodies), drives_of, "throughput", 60, 0,
                         edit_at=(30, lambda d: _breaks_mid_run(None, _first_new(None, held["d"]))(d)))
    assert broke_at == 30


def _conj(q):
    return np.array([-q[0], -q[1], -q[2], q[3]])


def _qmul(l, r):
    return np.append(l[3] * r[:3] + r[3] * l[:3] + np.cross(l[:3], r[:3]), l[3] * r[3] - l[:3] @ r[:3])


def _coordinates(j, xf):
    """(swing, twist, hinge angle, s) of joint j in float64 from the transforms, by the header's definitions."""
    a, b = int(j["a"]), int(j["b"])
    qa = xf["rotation"][a].astype(np.float64)
    qb = xf["rotation"][b].astype(np.float64) if b else np.array([0.0, 0.0, 0.0, 1.0])
    d = _qmul(_qmul(qa, j["rel_rotation"].astype(np.float64)), _conj(qb))
    d = -d if d[3] < 0 else d
    u = _quat_rotate(qa, j["axis_a"].astype(np.float64))
    a_ = d[:3] @ u
    swing = 2.0 * np.arctan2(np.linalg.norm(d[:3] - u * a_), np.hypot(a_, d[3]))
    twist = 2.0 * np.arctan2(-a_, d[3])
    wa = xf["position"][a].astype(np.float64) + _quat_rotate(qa, j["anchor_a"].astype(np.float64))
    wb = (xf["position"][b].astype(np.float64) + _quat_rotate(qb, j["anchor_b"].astype(np.float64))) if b else j["anchor_b"].astype(np.float64)
    return swing, twist, twist, (wb - wa) @ u, np.linalg.norm((wb - wa) - ((wb - wa) @ u) * u)


def _link(type_, a, b, at, xf, axis):
    """A joint between a and b (0: the world) at the world point `at`, at rest for the unrotated transforms xf."""
    j = np.zeros(1, nudge_b200.JOINT)[0]
    j["type"], j["a"], j["b"], j["beta"] = type_, a, b, 0.2
    j["anchor_a"] = np.float32(at) - xf["position"][a]
    j["anchor_b"] = np.float32(at) - (xf["position"][b] if b else 0.0)
    j["axis_a"] = j["axis_b"] = axis; j["rel_rotation"] = (0.0, 0.0, 0.0, 1.0)
    return j


def _mechanisms():
    """One scene: a ten-body ragdoll hanging from the world by its torso, spinning; a motorised piston; a sliding door thrown at its stop.
    The limbs reach to within 0.05 of their joints, and each slider's anchors sit where it comes to rest: a point or slider row whose lever
    arm is long against the body's size converges slowly under the solver's scalar sweeps (DESIGN.md section 8.20)."""
    s, _ = _free_bodies(12, 12)
    s.gravity = np.float32(9.82)
    xf = s.transforms
    size = {1: (0.2, 0.25, 0.1), 2: (0.1, 0.1, 0.1), 11: (0.3, 0.3, 0.3), 12: (0.5, 1.0, 0.05)}
    for k in range(1, 13):
        s.box_data["size"][k] = size.get(k, (0.25, 0.07, 0.07) if k in (3, 4, 5, 6) else (0.07, 0.25, 0.07))
    s.properties[1:] = scenes._box_props(s.box_data["size"][1:])
    s.momentum["velocity"][:] = 0.0; s.momentum["angular_velocity"][:] = 0.0
    xf["rotation"][:] = (0.0, 0.0, 0.0, 1.0)
    o = np.array([0.0, 500.0, 0.0], np.float32)
    at = {1: (0, 0, 0), 2: (0, 0.6, 0), 3: (0.6, 0.2, 0), 4: (-0.6, 0.2, 0), 5: (1.2, 0.2, 0), 6: (-1.2, 0.2, 0),
          7: (0.25, -0.6, 0), 8: (-0.25, -0.6, 0), 9: (0.25, -1.2, 0), 10: (-0.25, -1.2, 0), 11: (40, 0, 0), 12: (80, 0, 0)}
    for k, p in at.items():
        xf["position"][k] = o + np.float32(p)
    joints, drives = [_link(BALL, 1, 0, o, xf, (0, 1, 0))], []

    def drive(flags, **kw):
        d = np.zeros(1, nudge_b200.JOINT_DRIVE)[0]
        d["joint"], d["flags"], d["break_force"], d["break_torque"] = len(joints) - 1, flags, np.inf, np.inf
        for k, v in kw.items():
            d[k] = v
        drives.append(d)
    # neck, shoulders, hips: cone + twist about the limb; elbows and knees: hinge limits
    for child, parent, pivot, axis, cone, tw in ((2, 1, (0, 0.3, 0), (0, 1, 0), 0.5, 0.6), (3, 1, (0.3, 0.2, 0), (1, 0, 0), 1.2, 0.8),
                                                  (4, 1, (-0.3, 0.2, 0), (-1, 0, 0), 1.2, 0.8), (7, 1, (0.25, -0.3, 0), (0, -1, 0), 0.8, 0.4),
                                                  (8, 1, (-0.25, -0.3, 0), (0, -1, 0), 0.8, 0.4)):
        joints.append(_link(BALL, child, parent, o + np.float32(pivot), xf, axis))
        drive(CN | TW, cone=cone, lower=-tw, upper=tw)
    for child, parent, pivot, axis, lo, hi in ((5, 3, (0.9, 0.2, 0), (0, 0, 1), -1.0, 0.2), (6, 4, (-0.9, 0.2, 0), (0, 0, 1), -0.2, 1.0),
                                               (9, 7, (0.25, -0.9, 0), (1, 0, 0), -0.1, 1.5), (10, 8, (-0.25, -0.9, 0), (1, 0, 0), -0.1, 1.5)):
        joints.append(_link(HINGE, child, parent, o + np.float32(pivot), xf, axis))
        drive(L, lower=lo, upper=hi)
    # piston: s = -x travel, driven to its stop at 2; door: thrown along +x onto the stop at s = -1.  The anchors sit where the body
    # rests on its stop: anchor_a = the travel to the stop, anchor_b = the start plus that travel
    for body, travel, flags, kw in ((11, -2.0, S | L | M, dict(lower=-2.0, upper=2.0, motor_speed=1.5, max_motor_torque=50.0)),
                                    (12, 1.0, S | L, dict(lower=-1.0, upper=0.5))):
        joints.append(_link(FIXED, body, 0, xf["position"][body] + np.float32([travel, 0.0, 0.0]), xf, (1, 0, 0)))
        drive(flags, **kw)
    s.momentum["velocity"][12] = (3.0, 0.0, 0.0)
    rng = np.random.default_rng(4)
    s.momentum["angular_velocity"][2:11] = rng.normal(size=(9, 3)) * 2.0
    return s, np.array(joints), np.array(drives)


def test_ragdoll_piston_and_sliding_door_with_no_host_work_between_steps():
    s, joints, drives = _mechanisms()
    g = nudge_b200.Sim(s, stream=side_stream())
    g.upload_joints(joints); g.upload_joint_drives(drives)
    worst = np.zeros(len(drives))   # drive k is on joint k + 1
    piston_speed, door = [], []
    for step in range(240):
        g.step()
        g.download_bodies()
        assert np.isfinite(g.transforms["position"]).all() and np.isfinite(g.momentum["velocity"]).all()
        for i, (j, d) in enumerate(zip(joints[1:], drives)):
            swing, twist, angle, s_, off = _coordinates(j, g.transforms)
            f = int(d["flags"])
            if f & CN:
                worst[i] = max(worst[i], swing - d["cone"], twist - d["upper"], d["lower"] - twist)
            elif f & S:
                worst[i] = max(worst[i], s_ - d["upper"], d["lower"] - s_, off)
            elif f & L:
                worst[i] = max(worst[i], angle - d["upper"], d["lower"] - angle)
        if step == 40:
            piston_speed.append(-float(g.momentum["velocity"][11][0]))
        door.append(_coordinates(joints[11], g.transforms)[3])
    assert g.debug_scalar("graph_records") == 1
    # stated tolerances: 0.1 rad for the ragdoll's cones, twists and hinge stops under spin and gravity, 0.02 for the slider stops
    assert worst[:9].max() < 0.1, worst
    assert worst[9:].max() < 0.02, worst
    assert abs(piston_speed[0] - 1.5) < 0.01
    s_piston = _coordinates(joints[10], g.transforms)[3]
    assert abs(s_piston - 2.0) < 0.02 and abs(door[-1] + 1.0) < 0.02 and min(door) > -1.02
    back = g.download_joint_drives()
    assert abs(back[9]["position"] - s_piston) < 0.05 and (back["cone"][:5] == drives["cone"][:5]).all()


def _pile_with_dof(seed, m=40, stream=True):
    s = _pile()
    g = nudge_b200.Sim(s, stream=side_stream()) if stream else nudge_b200.Sim(s)
    rng = np.random.default_rng(seed)
    joints = _joints_at_rest(s.transforms, rng, m, s.n_bodies)
    drives = _dof_drives_on_all(joints, rng)
    g.upload_joints(joints); g.upload_joint_drives(drives)
    return s, g, joints, drives, rng


def test_new_cones_and_ranges_keep_the_graph_and_add_no_launch():
    s, g, joints, drives, rng = _pile_with_dof(8)
    per_step = []
    cone, slide = (drives["flags"] & CN) != 0, (drives["flags"] & S) != 0
    for step in range(100):
        drives["cone"][cone] = rng.uniform(0.2, 1.5, cone.sum())
        drives["lower"][slide] = -rng.uniform(0.1, 0.5, slide.sum())
        g.upload_joint_drives(drives)
        before = g.launch_count(); g.step(); per_step.append(g.launch_count() - before)
    assert g.debug_scalar("graph_records") == 1 and len(set(per_step)) == 1
    k = int(np.flatnonzero(cone)[0])
    drives[k]["flags"] = int(drives[k]["flags"]) & ~TW   # another structure: one new record
    g.upload_joint_drives(drives)
    for _ in range(3):
        g.step()
    assert g.debug_scalar("graph_records") == 2
    g.upload_joint_drives(None)
    before = g.launch_count(); g.step()
    assert g.launch_count() - before == per_step[0]


def test_snapshot_restore_repeats_a_run():
    s, g, joints, drives, rng = _pile_with_dof(6)
    for _ in range(10):
        g.step()
    snap = g.snapshot()

    def run():
        for _ in range(30):
            g.step()
        return _body_bytes(g) + g.download_joints().tobytes() + g.download_joint_drives().tobytes()
    first = run()
    g.restore(snap)
    assert run() == first
    assert g.debug_scalar("graph_records") == 1


def test_state_file_keeps_the_flags_and_cones(tmp_path):
    s, g, joints, drives, rng = _pile_with_dof(7, stream=False)
    h = nudge_b200.Sim(s)
    for _ in range(5):
        g.step()
    path = str(tmp_path / "dof.nbstate")
    g.save_state(path)
    h.load_state(path)
    a, b = g.download_joint_drives(), h.download_joint_drives()
    assert a["flags"].tobytes() == b["flags"].tobytes() == np.sort(drives, order="joint")["flags"].tobytes()
    assert a["cone"].tobytes() == b["cone"].tobytes() == np.sort(drives, order="joint")["cone"].tobytes()
    assert _without_position(a) == _without_position(b)
    for _ in range(5):
        g.step(); h.step()
    assert _body_bytes(g) == _body_bytes(h) and h.download_joint_drives().tobytes() == g.download_joint_drives().tobytes()


def test_body_removal_renumbers_the_new_drives():
    s, g, joints, drives, rng = _pile_with_dof(4, m=60, stream=False)
    for _ in range(3):
        g.step()
    before_j, before_d = g.download_joints(), g.download_joint_drives()
    gone = np.array([int(joints[5]["a"]), 57, 130], np.uint32)
    g.remove_bodies(gone)
    keep = ~(np.isin(before_j["a"], gone) | np.isin(before_j["b"], gone))
    new_index = np.cumsum(keep) - 1
    want = before_d[keep[before_d["joint"]]].copy()
    want["joint"] = new_index[want["joint"]]
    got = g.download_joint_drives()
    assert 0 < len(got) < len(before_d) and _without_position(got) == _without_position(want)
    assert (got["flags"] & (S | CN | TW)).any()
    for _ in range(3):
        g.step()
    g.download_bodies()
    assert np.isfinite(g.transforms["position"]).all()


def test_new_refusals_change_nothing():
    s, g, joints, drives, rng = _pile_with_dof(9, m=20, stream=False)
    kept = g.download_joint_drives().tobytes()
    types = joints["type"]
    ball, fixed = int(np.flatnonzero(types == BALL)[0]), int(np.flatnonzero(types == FIXED)[0])
    hinge = int(np.flatnonzero(types == HINGE)[0])

    def one(joint, flags, **kw):
        d = np.zeros(1, nudge_b200.JOINT_DRIVE); d["joint"], d["flags"] = joint, flags
        d["break_force"] = d["break_torque"] = np.inf
        for k, v in kw.items():
            d[k] = v
        return d
    cases = [(one(ball, CN, cone=0.0), r"cone outside \(0, pi\]"), (one(ball, CN, cone=3.2), r"cone outside \(0, pi\]"),
             (one(ball, CN, cone=np.nan), r"cone outside \(0, pi\]"), (one(ball, CN, cone=0.5, motor_speed=1.0), "motor speed or torque"),
             (one(ball, CN, cone=0.5, max_motor_torque=1.0), "motor speed or torque"), (one(ball, TW, lower=0.5, upper=0.2), "lower > upper"),
             (one(ball, TW, lower=-3.5, upper=0.0), r"twist limit outside \[-pi, pi\]"), (one(ball, TW, lower=0.0, upper=3.2), r"twist limit outside"),
             (one(hinge, S), "does not take"), (one(hinge, CN, cone=0.5), "does not take"), (one(fixed, TW), "does not take"),
             (one(fixed, L | M), "does not take"), (one(ball, S), "does not take"), (one(ball, M | CN, cone=0.5), "does not take"),
             (one(fixed, S | L, lower=1.0, upper=0.5), "lower > upper"), (one(hinge, 128), "unknown flag")]
    for d, what in cases:
        with pytest.raises(nudge_b200.NudgeError, match=what):
            g.upload_joint_drives(d)
        assert g.download_joint_drives().tobytes() == kept
    bent = joints.copy(); bent[ball]["axis_a"] = (0.0, 1.1, 0.0); bent[fixed]["axis_a"] = (0.0, 0.0, 0.9)
    g.upload_joints(bent)   # the same structure: the drives stay
    for d in (one(ball, CN, cone=0.5), one(ball, TW), one(fixed, S)):
        with pytest.raises(nudge_b200.NudgeError, match="axis_a is not of unit length"):
            g.upload_joint_drives(d)
    bent = joints.copy(); bent[ball]["rel_rotation"] = (0.0, 0.0, 0.0, 1.01)
    g.upload_joints(bent)
    for d in (one(ball, CN, cone=0.5), one(ball, TW)):
        with pytest.raises(nudge_b200.NudgeError, match="rel_rotation is not of unit length"):
            g.upload_joint_drives(d)
    assert g.download_joint_drives().tobytes() == kept
    g.upload_joint_drives(one(ball, BR, cone=np.nan, motor_speed=1.0))   # without CONE the cone is not read
    assert g.download_joint_drives()["cone"][0] == 0
    g.upload_joints(joints)
    g.upload_joint_drives(one(ball, CN | TW | BR, cone=np.float32(np.pi), lower=np.float32(-np.pi), upper=np.float32(np.pi)))
    g.upload_joint_drives(one(fixed, S | L | M | BR, lower=-1e6, upper=1e6))   # any finite range
    assert len(g.download_joint_drives()) == 1
