"""Joint drives (nb_upload_joint_drives, nb_download_joint_drives; DESIGN.md section 8.17): the drive rows and the device drive table byte
for byte against the numpy restatement (tests/joint_drives_ref.py); runs with drives byte for byte against a twin fed the restated rows through
nb_upload_constraint_rows, breaks included; a door, a wheel, a rope and a breaking weld under one graph record; the graph and launch rules;
snapshots, state files, body removal and joint uploads; and the refusals."""
import numpy as np
import pytest
import nudge_b200
from nudge_b200 import scenes
from oracle import joints_ref
from tests import joint_drives_ref as drives_ref
from tests.gpu_util import side_stream, joint_rows, STATE_HEADER
from tests.test_gpu_rows import _free_bodies, _pile
from tests.test_gpu_joints import _joints_at_rest, _body_bytes

pytestmark = pytest.mark.gpu
ROWS = joints_ref.ROWS_PER_TYPE
L, M, BR = drives_ref.LIMIT, drives_ref.MOTOR, drives_ref.BREAKABLE
TAKES = {joints_ref.BALL: BR, joints_ref.HINGE: L | M | BR, joints_ref.FIXED: BR, joints_ref.DISTANCE: L | BR}


def _random_drives(joints, rng, share=0.7, broken=0.0, fragile=0.0):
    """Drives on a random share of the joints with random flags their types take; `fragile` of them BREAKABLE with zero thresholds."""
    out = []
    for i, j in enumerate(joints):
        if rng.random() > share:
            continue
        t = int(j["type"])
        d = np.zeros(1, nudge_b200.JOINT_DRIVE)[0]
        d["joint"] = i
        d["flags"] = int(rng.integers(0, 8)) & TAKES[t]
        if t == joints_ref.HINGE:
            d["lower"], d["upper"] = np.sort(rng.uniform(-np.pi, np.pi, 2))
        else:
            d["lower"], d["upper"] = np.sort(rng.uniform(0.0, 3.0, 2))
        d["motor_speed"], d["max_motor_torque"] = rng.normal() * 2.0, rng.random() * 5.0
        d["break_force"], d["break_torque"] = (0.0, 0.0) if rng.random() < fragile else (np.inf, rng.random() * 50.0 if rng.random() < 0.5 else np.inf)
        d["impulse"] = rng.normal(size=3) * 0.01
        d["broken"] = 1 if rng.random() < broken else 0
        out.append(d)
    return np.array(out, nudge_b200.JOINT_DRIVE)


def _drive_impulses(joints, table, imp, driven):
    """The impulse[3] (motor, lower, upper) of the drives on the joints `driven`, from the appended rows' impulses in joint order."""
    out, m = {}, 0
    for i in range(len(joints)):
        fl = int(table["flags"][i])
        v = np.zeros(3, np.float32)
        for k in range(3):
            if fl & (L if k else M):
                v[k] = imp[m]; m += 1
        out[i] = v
    return np.array([out[i] for i in driven], np.float32).reshape(-1, 3)


def test_own_rows_drive_rows_and_table_equal_the_numpy_restatement_byte_for_byte():
    n = 60
    s, rng = _free_bodies(n, 4)
    g = nudge_b200.Sim(s)
    m = 320
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
    joints[9]["type"], joints[9]["a"], joints[9]["b"] = joints_ref.DISTANCE, 3, 0   # coinciding anchors: the fallback direction
    joints[9]["anchor_a"] = 0.0; joints[9]["anchor_b"] = s.transforms["position"][3]
    drives = _random_drives(joints, rng, broken=0.05, fragile=0.1)
    g.upload_joints(joints); g.upload_joint_drives(drives)
    order = joints_ref.table_order(joints)
    table = g.debug("joint_drives", drives_ref.DRIVE_TABLE)
    before = joint_rows(g)
    n_own = int(sum(ROWS[t] for t in joints["type"]))
    # the upload: the host's table and the uploaded impulses, in table order
    want_table, want_imp = drives_ref.drive_table(joints[order], _renumber(drives, order))
    assert table.tobytes() == want_table.tobytes()
    assert before["impulse"][n_own:].tobytes() == want_imp.tobytes()
    g.collide(); g.apply_gravity_damping(); g.read_cached_impulses(); g.setup_contact_constraints()
    got = joint_rows(g)
    g.download_bodies()
    dt = np.float32(s.time_step)
    jt = joints[order]
    table["broken"] = drives_ref.broken_after(jt, before, table, dt)
    assert 0 < table["broken"].sum() < len(drives)
    want = drives_ref.joint_rows(jt, g.transforms, dt, table, before["impulse"][n_own:])
    assert len(got) == len(want) == n_own + sum(drives_ref.drive_row_count(int(f)) for f in drives["flags"])
    for k in nudge_b200.ROW.names:
        assert got[k].tobytes() == want[k].tobytes(), k
    assert g.debug("joint_drives", drives_ref.DRIVE_TABLE).tobytes() == table.tobytes()
    g.apply_impulses(int(s.iterations)); g.update_cached_impulses(); g.write_cached_impulses(); g.advance()
    back = g.download_joint_drives()
    assert list(back["joint"]) == sorted(drives["joint"])
    for k in ("flags", "lower", "upper", "motor_speed", "max_motor_torque", "break_force", "break_torque"):
        assert back[k].tobytes() == np.sort(drives, order="joint")[k].tobytes(), k
    assert np.isfinite(back["impulse"]).all() and (back["broken"] == table["broken"][np.argsort(order)][back["joint"]]).all()


def _renumber(drives, order):
    """The drives with joint = the joint's position in `order`."""
    pos = np.argsort(order)
    d = drives.copy(); d["joint"] = pos[drives["joint"]]
    return d


def _twin_run(s, joints_of, drives_of, mode, steps, settle, edit_at=None):
    """x runs with joints and drives; y gets the restated rows (joint order: own rows, then the drive's) through nb_upload_constraint_rows,
    with the break rule applied from its downloaded impulses.  At `edit_at` a new drive list (edit(download)) goes to both."""
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
    table, imp = drives_ref.drive_table(yj, drives)
    order = drives_ref.solve_order(yj, table)
    n_own = int(sum(ROWS[t] for t in joints["type"]))
    dt = np.float32(s.time_step)
    prev, broke_at = None, None
    for step in range(steps):
        if edit_at and step == edit_at[0]:
            drives = edit_at[1](x.download_joint_drives())
            x.upload_joint_drives(drives)
            table, imp = drives_ref.drive_table(yj, drives)   # the same rows with the same impulses: prev stays what the break test reads
            order = drives_ref.solve_order(yj, table)
        if prev is not None:
            table["broken"] = drives_ref.broken_after(yj, prev, table, dt)
        y.download_bodies()
        rows = drives_ref.joint_rows(yj, y.transforms, dt, table, imp)
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
    return broke_at, x


def _breaks_mid_run(joints, first):
    """An edit that gives joint `first`'s BREAKABLE drive thresholds 0: it breaks at the next build."""
    def edit(d):
        d = d.copy()
        k = int(np.flatnonzero(d["joint"] == first)[0])
        d[k]["break_force"] = 0.0; d[k]["break_torque"] = 0.0
        return d
    return edit


def _drives_on_all(joints, rng):
    d = _random_drives(joints, rng, share=1.0)
    d["break_force"] = np.inf; d["break_torque"] = np.inf; d["broken"] = 0
    d["flags"] = [int(f) | BR | (L if TAKES[int(joints[int(i)]["type"])] & L else 0) for f, i in zip(d["flags"], d["joint"])]
    return d


def test_drives_equal_the_row_path_among_contacts_in_parity_mode():
    s = _pile()
    rng = np.random.default_rng(3)
    holder = {}
    broke_at, _ = _twin_run(s, lambda xf: holder.setdefault("j", _joints_at_rest(xf, rng, 48, s.n_bodies)), lambda j: _drives_on_all(j, rng),
                            "parity", 60, 30, edit_at=(25, lambda d: _breaks_mid_run(holder["j"], 0)(d)))
    assert broke_at == 25


def test_drives_equal_the_row_path_in_throughput_mode_without_contacts():
    s, rng = _free_bodies(40, 5)
    holder = {}
    broke_at, _ = _twin_run(s, lambda xf: holder.setdefault("j", _joints_at_rest(xf, rng, 36, s.n_bodies)), lambda j: _drives_on_all(j, rng),
                            "throughput", 60, 0, edit_at=(30, lambda d: _breaks_mid_run(holder["j"], 1)(d)))
    assert broke_at == 30


def _world_hinge(xf, a, anchor_local, axis=(0.0, 0.0, 1.0)):
    j = np.zeros(1, nudge_b200.JOINT)[0]
    j["type"], j["a"], j["b"], j["beta"] = joints_ref.HINGE, a, 0, 0.2
    j["anchor_a"] = anchor_local; j["anchor_b"] = xf["position"][a] + np.float32(anchor_local)
    j["axis_a"] = j["axis_b"] = axis; j["rel_rotation"] = (0.0, 0.0, 0.0, 1.0)
    return j


def test_door_wheel_rope_and_breaking_weld_with_no_host_work_between_steps():
    s, _ = _free_bodies(8, 12)
    s.gravity = np.float32(9.82)
    xf = s.transforms
    s.box_data["size"][1:] = (0.5, 0.5, 0.5)
    s.properties[1:] = scenes._box_props(s.box_data["size"][1:])
    s.momentum["velocity"][:] = 0.0; s.momentum["angular_velocity"][:] = 0.0
    xf["rotation"][:] = (0.0, 0.0, 0.0, 1.0)
    for k in range(1, 9):
        xf["position"][k] = (20.0 * k, 500.0, 0.0)
    door, wheel = _world_hinge(xf, 1, (-1.0, 0.0, 0.0)), _world_hinge(xf, 2, (0.0, 0.0, 0.0))
    rope = np.zeros(1, nudge_b200.JOINT)[0]
    rope["type"], rope["a"], rope["beta"], rope["length"], rope["rel_rotation"] = joints_ref.DISTANCE, 3, 0.2, 1.0, (0, 0, 0, 1)
    rope["anchor_b"] = xf["position"][3] + np.float32([0.0, 1.0, 0.0])
    welds = []
    for a in (4, 5):
        w = np.zeros(1, nudge_b200.JOINT)[0]
        w["type"], w["a"], w["beta"], w["rel_rotation"] = joints_ref.FIXED, a, 0.2, (0, 0, 0, 1)
        w["anchor_b"] = xf["position"][a]
        welds.append(w)
    joints = np.array([door, wheel, rope] + welds)
    mass = 1.0 / float(s.properties["mass_inverse"][4])
    load = mass * float(s.gravity)
    drives = np.zeros(5, nudge_b200.JOINT_DRIVE)
    drives["joint"] = np.arange(5); drives["break_force"] = np.inf; drives["break_torque"] = np.inf
    drives[0]["flags"], drives[0]["lower"], drives[0]["upper"] = L, -0.3, 0.5
    drives[1]["flags"], drives[1]["motor_speed"], drives[1]["max_motor_torque"] = M, 4.0, 500.0
    drives[2]["flags"], drives[2]["lower"], drives[2]["upper"] = L, 0.0, 2.0
    drives[3]["flags"], drives[3]["break_force"] = BR, 0.5 * load
    drives[4]["flags"], drives[4]["break_force"] = BR, 2.5 * load
    g = nudge_b200.Sim(s, stream=side_stream())
    g.upload_joints(joints); g.upload_joint_drives(drives)
    hinge0 = xf["position"][1].astype(np.float64) + (-1.0, 0.0, 0.0)
    thetas = []
    for step in range(240):
        g.step()
        if step % 4 == 3:
            g.download_bodies()
            p = g.transforms["position"][1].astype(np.float64) - hinge0
            thetas.append(-np.arctan2(p[1], p[0]))
    assert g.debug_scalar("graph_records") == 1
    g.download_bodies()
    p = g.transforms["position"].astype(np.float64)
    assert -0.33 < min(thetas) and max(thetas) < 0.53 and abs(thetas[-1] - 0.5) < 0.03, (min(thetas), max(thetas))   # the door rests on its stop
    assert abs(-float(g.momentum["angular_velocity"][2][2]) - 4.0) < 0.05                                               # the wheel turns at its speed
    assert abs(np.linalg.norm(p[3] - rope["anchor_b"]) - 2.0) < 0.05                                                    # the rope hangs at its length
    d = g.download_joint_drives()
    assert list(d["broken"]) == [0, 0, 0, 1, 0]
    assert p[4][1] < 490.0 and abs(p[5][1] - 500.0) < 0.05                                                              # one weld gave way
    assert abs(d[0]["position"] - thetas[-1]) < 0.03 and abs(d[2]["position"] - 2.0) < 0.05


def _pile_with_drives(seed, m=40, stream=True):
    s = _pile()
    g = nudge_b200.Sim(s, stream=side_stream()) if stream else nudge_b200.Sim(s)
    rng = np.random.default_rng(seed)
    joints = _joints_at_rest(s.transforms, rng, m, s.n_bodies)
    drives = _drives_on_all(joints, rng)
    g.upload_joints(joints); g.upload_joint_drives(drives)
    return s, g, joints, drives, rng


def test_throttle_keeps_the_graph_and_drives_add_no_launch():
    s, g, joints, drives, rng = _pile_with_drives(8)
    per_step = []
    for step in range(100):
        drives["motor_speed"] = rng.normal(size=len(drives))
        g.upload_joint_drives(drives)
        before = g.launch_count(); g.step(); per_step.append(g.launch_count() - before)
    assert g.debug_scalar("graph_records") == 1 and len(set(per_step)) == 1
    drives[0]["flags"] ^= M if TAKES[int(joints[int(drives[0]["joint"])]["type"])] & M else BR   # another structure: one new record
    g.upload_joint_drives(drives)
    for _ in range(3):
        g.step()
    assert g.debug_scalar("graph_records") == 2
    g.upload_joint_drives(None)
    before = g.launch_count(); g.step()
    assert g.launch_count() - before == per_step[0] and len(g.download_joint_drives()) == 0
    assert len(joint_rows(g)) == sum(ROWS[t] for t in joints["type"])


def test_snapshot_restore_repeats_a_run_with_a_break():
    s, g, joints, drives, rng = _pile_with_drives(6)
    for _ in range(10):
        g.step()
    snap = g.snapshot()
    d = g.download_joint_drives()
    d[3]["break_force"] = 0.0; d[3]["break_torque"] = 0.0   # every drive is BREAKABLE already: the same structure
    records = g.debug_scalar("graph_records")

    def run():
        g.upload_joint_drives(d)
        for _ in range(30):
            g.step()
        return _body_bytes(g) + g.download_joints().tobytes() + g.download_joint_drives().tobytes()
    first = run()
    assert g.download_joint_drives()["broken"][3] == 1
    g.restore(snap)
    assert g.download_joint_drives()["broken"].sum() == 0
    assert run() == first
    assert g.debug_scalar("graph_records") == records == 1   # new thresholds, a break and the restore all keep the graph


def _without_position(d):
    d = d.copy(); d["position"] = 0
    return d.tobytes()


def test_state_file_version_7_round_trip_and_a_version_6_file(tmp_path):
    s, g, joints, drives, rng = _pile_with_drives(7, stream=False)
    h, plain = nudge_b200.Sim(s), nudge_b200.Sim(s)
    plain.upload_joints(joints)
    for _ in range(5):
        g.step()
    new, v6 = str(tmp_path / "new.nbstate"), str(tmp_path / "v6.nbstate")
    g.save_state(new); plain.save_state(v6)
    head = STATE_HEADER.unpack(open(new, "rb").read(STATE_HEADER.size))
    assert head[1] == 7 and head[8 + 6] == len(joints) and head[8 + 7] == len(drives)
    assert STATE_HEADER.unpack(open(v6, "rb").read(STATE_HEADER.size))[1] == 6
    h.load_state(new)
    assert _without_position(h.download_joint_drives()) == _without_position(g.download_joint_drives())
    for _ in range(5):
        g.step(); h.step()
    assert _body_bytes(g) == _body_bytes(h) and h.download_joint_drives().tobytes() == g.download_joint_drives().tobytes()
    g.load_state(v6)
    assert len(g.download_joint_drives()) == 0 and len(g.download_joints()) == len(joints)


def test_body_removal_renumbers_drives_and_joint_uploads_keep_or_drop_them():
    s, g, joints, drives, rng = _pile_with_drives(4, m=60, stream=False)
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
    # nb_upload_joints: the same structure keeps the drives with their impulses and broken flags, another removes them
    d = g.download_joint_drives(); d[0]["broken"] = 1
    g.upload_joint_drives(d)
    kept = g.download_joint_drives()
    tuned = g.download_joints(); tuned["beta"] = 0.1
    g.upload_joints(tuned)
    assert g.download_joint_drives().tobytes() == kept.tobytes() and kept["broken"][0] == 1
    g.upload_joints(tuned[:-1])
    assert len(g.download_joint_drives()) == 0
    for _ in range(3):
        g.step()
    g.download_bodies()
    assert np.isfinite(g.transforms["position"]).all()


def test_refusals_change_nothing():
    s, g, joints, drives, rng = _pile_with_drives(9, m=20, stream=False)
    kept = g.download_joint_drives().tobytes()
    types = joints["type"]
    hinge = int(np.flatnonzero(types == joints_ref.HINGE)[0]); dist = int(np.flatnonzero(types == joints_ref.DISTANCE)[0])
    ball = int(np.flatnonzero(types == joints_ref.BALL)[0])

    def one(joint, flags, **kw):
        d = np.zeros(1, nudge_b200.JOINT_DRIVE); d["joint"], d["flags"] = joint, flags
        d["break_force"] = d["break_torque"] = np.inf
        for k, v in kw.items():
            d[k] = v
        return d
    cases = [(one(len(joints), BR), "beyond the joint count"), (np.concatenate([one(ball, BR), one(ball, BR)]), "two drives"),
             (one(ball, L), "does not take"), (one(dist, M), "does not take"), (one(hinge, 8), "unknown flag"),
             (one(hinge, L, lower=0.5, upper=0.2), "lower > upper"), (one(hinge, L, lower=-3.5, upper=0.0), r"\[-pi, pi\]"),
             (one(hinge, L, lower=0.0, upper=3.2), r"\[-pi, pi\]"), (one(dist, L, lower=-0.1, upper=1.0), "negative distance"),
             (one(hinge, M, max_motor_torque=-1.0), "negative"), (one(ball, BR, break_force=-1.0), "negative"),
             (one(ball, BR, break_torque=-np.inf), "threshold"), (one(ball, BR, break_force=np.nan), "threshold"),
             (one(hinge, M, motor_speed=np.inf), "not finite"), (one(hinge, L, impulse=(0.0, np.nan, 0.0)), "not finite"),
             (one(ball, BR, broken=2), "broken")]
    for d, what in cases:
        with pytest.raises(nudge_b200.NudgeError, match=what):
            g.upload_joint_drives(d)
        assert g.download_joint_drives().tobytes() == kept
    assert g.lib.nb_upload_joint_drives(g.ctx, None, 3, g.stream) == -3   # NB_ERR_ARGUMENT
    # a HINGE LIMIT needs a unit rel_rotation; float32(pi) is inside the range
    bent = joints.copy(); bent[hinge]["rel_rotation"] = (0.0, 0.0, 0.0, 1.01)
    g.upload_joints(bent)   # the same structure: the drives stay
    with pytest.raises(nudge_b200.NudgeError, match="unit length"):
        g.upload_joint_drives(one(hinge, L, lower=-1.0, upper=1.0))
    assert g.download_joint_drives().tobytes() == kept
    g.upload_joint_drives(one(hinge, M | BR))   # without LIMIT the rest pose is not read
    g.upload_joints(joints)
    g.upload_joint_drives(one(hinge, L | M | BR, lower=np.float32(-np.pi), upper=np.float32(np.pi)))
    assert len(g.download_joint_drives()) == 1
