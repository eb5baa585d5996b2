"""Device-resident joints (nb_upload_joints, nb_download_joints; DESIGN.md section 8.13): the generated rows byte for byte against the numpy
restatement (oracle/joints_ref.py); a jointed run byte for byte against the same run fed through nb_upload_constraint_rows from the host
every step; physical checks of the four types with no host work between steps; graph replay; the launch arithmetic; spawning, snapshots,
state files; and the refusals."""
import numpy as np
import pytest
import nudge_b200
from nudge_b200 import scenes
from oracle import joints_ref
from tests.gpu_util import side_stream, STATE_HEADER
from tests.test_gpu_rows import _free_bodies, _pile, _quat_rotate, _quat_unrotate
from tests.test_joints_ref import _errors, _qmul

pytestmark = pytest.mark.gpu
ROWS = joints_ref.ROWS_PER_TYPE


def _conj(q):
    return np.array([-q[0], -q[1], -q[2], q[3]])


def _at_rest(xf, type_, a, b, rng, softness=0.0, mid=False):
    """A joint between bodies a and b (0: the world) with no error at the transforms xf: the anchor at a's centre, or midway between the two."""
    j = np.zeros(1, nudge_b200.JOINT)[0]
    pa, qa = xf["position"][a].astype(np.float64), xf["rotation"][a].astype(np.float64)
    pb, qb = (xf["position"][b].astype(np.float64), xf["rotation"][b].astype(np.float64)) if b else (np.zeros(3), np.array([0.0, 0.0, 0.0, 1.0]))
    axis = rng.normal(size=3); axis /= np.linalg.norm(axis)
    j["type"], j["a"], j["b"], j["beta"], j["softness"] = type_, a, b, 0.2, softness
    at = 0.5 * (pa + pb) if mid else pa
    j["anchor_a"] = _quat_unrotate(qa, at - pa); j["anchor_b"] = _quat_unrotate(qb, at - pb)
    j["axis_a"] = axis; j["axis_b"] = _quat_unrotate(qb, _quat_rotate(qa, axis))
    j["rel_rotation"] = _qmul(_conj(qa), qb)
    if type_ == joints_ref.DISTANCE:   # a rod of random length from a's centre
        j["anchor_b"] = _quat_unrotate(qb, pa + rng.normal(size=3) - pb)
        wb = pb + _quat_rotate(qb, j["anchor_b"].astype(np.float64))
        j["length"] = np.linalg.norm(pa - wb)
    return j


def _joints_at_rest(xf, rng, m, n_bodies, world=0.2):
    out = []
    for i in range(m):
        a = int(rng.integers(1, n_bodies))
        b = 0 if rng.random() < world else int(rng.integers(1, n_bodies))
        if b == a:
            b = a % (n_bodies - 1) + 1
        out.append(_at_rest(xf, i % 4, a, b, rng, softness=0.01 if i % 3 == 0 else 0.0))
    return np.array(out)


def _body_bytes(g):
    g.download_bodies()
    return g.transforms.tobytes() + g.momentum.tobytes()


def test_generated_rows_equal_the_numpy_restatement_byte_for_byte():
    n = 60
    s, rng = _free_bodies(n, 4)
    g = nudge_b200.Sim(s)
    g.upload_kinematic_bodies(np.array([(k, (0.1, 0.0, 0.0), (0.0, 0.2, 0.0), 0) for k in (5, 17, 40)], scenes.KINEMATIC))
    m = 320
    joints = np.zeros(m, nudge_b200.JOINT)
    joints["type"] = rng.integers(0, 4, m); joints["a"] = rng.integers(1, n + 1, m); joints["b"] = rng.integers(0, n + 1, m)
    same = joints["a"] == joints["b"]; joints["b"][same] = joints["a"][same] % n + 1
    for k in ("anchor_a", "anchor_b"):
        joints[k] = rng.normal(size=(m, 3))
    for k in ("axis_a", "axis_b"):
        v = rng.normal(size=(m, 3)); joints[k] = v / np.linalg.norm(v, axis=1, keepdims=True)
    joints["axis_a"][:8] = np.eye(3)[[0, 1, 2, 0, 1, 2, 0, 1]]   # both branches of the perpendicular rule
    joints["rel_rotation"] = scenes._random_unit_quaternions(rng, m)
    joints["length"] = rng.random(m) * 3.0; joints["beta"] = 0.1 + 0.2 * rng.random(m); joints["softness"] = np.where(rng.random(m) < 0.5, 0.01, 0.0)
    joints["impulse"] = rng.normal(size=(m, 6)) * 0.1
    joints[9]["type"], joints[9]["a"], joints[9]["b"] = joints_ref.DISTANCE, 3, 0   # coinciding anchors: the fallback direction
    joints[9]["anchor_a"] = 0.0; joints[9]["anchor_b"] = s.transforms["position"][3]
    g.upload_joints(joints)
    g.collide(); g.apply_gravity_damping(); g.read_cached_impulses(); g.setup_contact_constraints()
    got = g.debug("joint_rows", nudge_b200.ROW)
    g.download_bodies()
    want = joints_ref.joint_rows(joints[joints_ref.table_order(joints)], g.transforms, np.float32(s.time_step))
    assert len(got) == len(want) == sum(ROWS[t] for t in joints["type"])
    for k in nudge_b200.ROW.names:
        assert got[k].tobytes() == want[k].tobytes(), k
    g.apply_impulses(int(s.iterations)); g.update_cached_impulses(); g.write_cached_impulses(); g.advance()
    g.download_bodies()
    assert np.isfinite(g.momentum["velocity"]).all()
    # the download: upload order, the parameters as uploaded, unused impulse slots zero
    back = g.download_joints()
    for k in nudge_b200.JOINT.names:
        if k != "impulse":
            assert back[k].tobytes() == joints[k].tobytes(), k
    unused = np.arange(6)[None, :] >= np.array(ROWS)[joints["type"]][:, None]
    assert (back["impulse"][unused] == 0).all() and np.isfinite(back["impulse"]).all()


def _against_the_row_path(s, joints, mode, steps, settle):
    x, y = nudge_b200.Sim(s), nudge_b200.Sim(s)
    for g in (x, y):
        g.set_solver_mode(mode)
        for _ in range(settle):
            g.step_staged()
    y.download_bodies()
    joints = joints(y.transforms)
    x.upload_joints(joints)
    yj = joints.copy()
    n_rows = sum(ROWS[t] for t in joints["type"])
    for step in range(steps):
        y.download_bodies()
        y.upload_constraint_rows(joints_ref.joint_rows(yj, y.transforms, np.float32(s.time_step)))
        x.step_staged(); y.step_staged()
        rows = y.download_constraint_rows(n_rows)
        joints_ref.set_impulses(yj, rows)
        xi = x.download_joints()["impulse"]
        x.download_bodies(); y.download_bodies()
        assert x.momentum.tobytes() == y.momentum.tobytes(), step
        assert x.transforms.tobytes() == y.transforms.tobytes(), step
        assert xi.tobytes() == yj["impulse"].tobytes(), step
    assert np.isfinite(x.transforms["position"]).all() and np.abs(xi).max() > 0


def test_jointed_run_equals_the_row_path_among_contacts_in_parity_mode():
    s = _pile()
    rng = np.random.default_rng(3)
    _against_the_row_path(s, lambda xf: _joints_at_rest(xf, rng, 48, s.n_bodies), "parity", 60, 30)


def test_jointed_run_equals_the_row_path_in_throughput_mode_without_contacts():
    s, rng = _free_bodies(40, 5)
    _against_the_row_path(s, lambda xf: _joints_at_rest(xf, rng, 36, s.n_bodies), "throughput", 60, 0)


def _chain_scene(links=10):
    s = scenes.demo_scene(links + 60, 0, iterations=12, spread=3.0, height=6.0, seed=5)
    s.box_data["size"][1:links + 1] = (0.2, 0.5, 0.2)
    s.properties[1:links + 1] = scenes._box_props(s.box_data["size"][1:links + 1])
    top = np.array([6.0, 8.0, 0.0])
    for k in range(links):
        s.transforms["position"][1 + k] = top + np.array([0.5 + 1.0 * k, 0.0, 0.0])
        s.transforms["rotation"][1 + k] = (0.0, 0.0, np.sin(np.pi / 4), np.cos(np.pi / 4))
    s.connections = np.zeros(links - 1, scenes.PAIR32); s.connections["a"] = 1 + np.arange(links - 1); s.connections["b"] = 2 + np.arange(links - 1)
    joints = np.zeros(links, nudge_b200.JOINT)
    joints["type"] = joints_ref.BALL; joints["beta"] = 0.2; joints["rel_rotation"][:, 3] = 1.0
    joints["a"] = 1 + np.arange(links); joints["b"] = np.arange(links)
    joints["anchor_a"] = (0.0, 0.5, 0.0); joints["anchor_b"] = (0.0, -0.5, 0.0); joints[0]["anchor_b"] = top
    return s, joints, top


def test_hanging_chain_driven_by_joints_with_no_host_work_between_steps():
    """The hanging chain of the row tests, its ten ball joints resident: 240 graph replays and nothing else."""
    links = 10
    s, joints, top = _chain_scene(links)
    g = nudge_b200.Sim(s, stream=side_stream())
    g.upload_joints(joints)
    worst = 0.0
    for step in range(240):
        g.step()
        if step > 20 and step % 8 == 0:
            g.download_bodies()
            worst = max([worst] + [_errors(j, g.transforms)[0] for j in joints[1:]])
    assert g.debug_scalar("graph_records") == 1
    assert worst < 0.08, worst
    g.download_bodies()
    assert np.isfinite(g.transforms["position"]).all() and g.counts().overflow == 0
    assert g.transforms["position"][links][1] < top[1] - 0.5 * links


def test_hinge_fixed_and_distance_joints_hold_their_errors():
    """A door on a world hinge, a welded pair and a rod, each thrown about: position and angular errors stay bounded, and the door still turns."""
    s, rng = _free_bodies(12, 12)
    xf = s.transforms
    s.box_data["size"][1:] = (0.3, 0.3, 0.3)   # small enough that the jointed pairs never touch
    s.properties[1:] = scenes._box_props(s.box_data["size"][1:])
    for k in range(1, 13):   # far from each other, but each jointed pair (2, 3), (4, 5), (7, 8) 1.5 apart
        xf["position"][k] = (20.0 * k, 500.0, 0.0)
    for a, b in ((2, 3), (4, 5), (7, 8)):
        xf["position"][b] = xf["position"][a] + np.float32([0.0, 1.5, 0.0])
    joints = np.array([_at_rest(xf, joints_ref.HINGE, 1, 0, rng), _at_rest(xf, joints_ref.HINGE, 2, 3, rng, mid=True), _at_rest(xf, joints_ref.FIXED, 4, 5, rng, mid=True),
                       _at_rest(xf, joints_ref.FIXED, 6, 0, rng), _at_rest(xf, joints_ref.DISTANCE, 7, 8, rng), _at_rest(xf, joints_ref.DISTANCE, 9, 0, rng)])
    u0 = _quat_rotate(xf["rotation"][1].astype(np.float64), joints[0]["axis_a"].astype(np.float64))
    s.momentum["angular_velocity"][1] = 2.0 * u0 + np.cross(u0, (0.3, 0.5, 0.7))
    g = nudge_b200.Sim(s, stream=side_stream())
    g.upload_joints(joints)
    worst = np.zeros((len(joints), 2))
    for step in range(180):
        g.step()
        if step > 30 and step % 6 == 0:   # once the initial relative velocities are absorbed
            g.download_bodies()
            worst = np.maximum(worst, [_errors(j, g.transforms) for j in joints])
    assert worst[:, 0].max() < 0.1 and worst[:, 1].max() < 0.15, worst
    g.download_bodies()
    w = g.momentum["angular_velocity"][1].astype(np.float64)
    u = _quat_rotate(g.transforms["rotation"][1].astype(np.float64), joints[0]["axis_a"].astype(np.float64))
    assert abs(w @ u) > 0.05 and np.linalg.norm(np.cross(w, u)) < 0.1 * np.linalg.norm(w) + 0.05   # it spins about its hinge axis only
    assert np.abs(g.momentum["velocity"][6]).max() < 0.05                                          # welded to the world


def test_graph_replay_equals_the_staged_calls_and_records_once():
    s = _pile()
    x, y = nudge_b200.Sim(s, stream=side_stream()), nudge_b200.Sim(s)
    rng = np.random.default_rng(8)
    joints = _joints_at_rest(s.transforms, rng, 40, s.n_bodies)
    rows = np.zeros(6, nudge_b200.ROW)   # user rows next to the joints: they run first
    rows["a"] = (3, 9, 3, 40, 41, 9); rows["lin_a"] = rng.normal(size=(6, 3)); rows["lo"], rows["hi"] = -np.inf, np.inf; rows["bias"] = 0.1
    for g in (x, y):
        g.upload_joints(joints); g.upload_constraint_rows(rows)
    per_step = []
    for step in range(100):
        before = x.launch_count()
        x.step(); y.step_staged()
        per_step.append(x.launch_count() - before)
        if step % 10 == 9:
            assert _body_bytes(x) == _body_bytes(y), step
            assert x.download_joints().tobytes() == y.download_joints().tobytes(), step
    assert x.debug_scalar("graph_active") == 1 and x.debug_scalar("graph_records") == 1
    assert len(set(per_step)) == 1
    # new parameters and impulses for the same structure keep the graph; another structure re-records it
    tuned = x.download_joints(); tuned["beta"] = 0.1; tuned["softness"] = 0.02
    for g in (x, y):
        g.upload_joints(tuned)
    for _ in range(5):
        x.step(); y.step_staged()
    assert x.debug_scalar("graph_records") == 1 and _body_bytes(x) == _body_bytes(y)
    x.upload_joints(tuned[:-1]); x.step()
    assert x.debug_scalar("graph_records") == 2


@pytest.mark.parametrize("mode", ["parity", "throughput"])
def test_joints_add_one_launch_plus_one_per_level_and_pass(mode):
    s = _pile()
    g = nudge_b200.Sim(s)
    g.set_solver_mode(mode)
    inert = np.zeros(1, nudge_b200.ROW); inert["a"] = 1   # one user row: the step already runs one sweep per solver launch
    g.upload_constraint_rows(inert)

    def launches():
        before = g.launch_count(); g.step(); return g.launch_count() - before
    base = launches()
    rng = np.random.default_rng(2)
    joints = _joints_at_rest(s.transforms, rng, 30, s.n_bodies)
    levels = int(joints_ref.joint_levels(joints).max()) + 1
    assert levels > 1
    g.upload_joints(joints)
    assert launches() == base + 1 + levels * (int(s.iterations) + 1)
    g.upload_joints(None)
    assert launches() == base and len(g.download_joints()) == 0
    # joints alone split the sweeps exactly as user rows do: the inert row then adds its one level per pass and nothing else
    g.upload_constraint_rows(np.zeros(0, nudge_b200.ROW))
    plain = launches()
    g.upload_joints(joints)
    alone = launches()
    g.upload_constraint_rows(inert)
    assert launches() == alone + int(s.iterations) + 1
    g.upload_joints(None); g.upload_constraint_rows(np.zeros(0, nudge_b200.ROW))
    assert launches() == plain


def test_remove_and_add_bodies_edit_the_joints_like_the_host():
    s = _pile()
    s.idle[:] = 200
    g = nudge_b200.Sim(s, max_bodies=s.n_bodies + 4, max_boxes=s.n_boxes + 4)
    rng = np.random.default_rng(4)
    joints = _joints_at_rest(s.transforms, rng, 60, s.n_bodies)
    joints["impulse"] = rng.normal(size=(60, 6)) * 0.01
    joints[0]["a"], joints[0]["b"], joints[1]["a"], joints[1]["b"] = 20, 21, 22, 20   # two joints that lose body 20
    g.upload_joints(joints)
    before = g.download_joints()
    gone = np.array([20, 57, 130], np.uint32)
    g.remove_bodies(gone)
    keep = ~(np.isin(before["a"], gone) | np.isin(before["b"], gone))
    assert 0 < keep.sum() < 59
    want = before[keep].copy()
    for k in ("a", "b"):
        want[k] = want[k] - np.searchsorted(gone, want[k])
    got = g.download_joints()
    assert got.tobytes() == want.tobytes()
    # the kept bodies on the other side of the deleted joints are awake, nobody else
    other = np.concatenate([before["b"][~keep & np.isin(before["a"], gone)], before["a"][~keep & np.isin(before["b"], gone)]])
    other = other[(other != 0) & ~np.isin(other, gone)]
    other = np.unique(other - np.searchsorted(gone, other))
    assert {20, 21} <= set(int(v) for v in other)   # 21 and 22 before the removal
    g.download_bodies()
    awake = np.flatnonzero(g.idle == 0)
    assert sorted(awake) == sorted(other)
    # adding bodies leaves the joints alone
    g.add_bodies(scenes.fragment([(0.0, 40.0, 0.0), (3.0, 40.0, 0.0)], first_tag=100000))
    assert g.download_joints().tobytes() == want.tobytes()
    for _ in range(3):
        g.step()
    g.download_bodies()
    assert np.isfinite(g.transforms["position"]).all()


def test_snapshot_restore_repeats_a_jointed_run_byte_for_byte():
    s = _pile()
    g = nudge_b200.Sim(s, stream=side_stream())
    rng = np.random.default_rng(6)
    g.upload_joints(_joints_at_rest(s.transforms, rng, 50, s.n_bodies))
    for _ in range(10):
        g.step()
    snap = g.snapshot()
    for _ in range(30):
        g.step()
    first = _body_bytes(g) + g.download_joints().tobytes()
    g.restore(snap)
    for _ in range(30):
        g.step()
    assert _body_bytes(g) + g.download_joints().tobytes() == first
    assert g.debug_scalar("graph_records") == 1
    # a snapshot taken without joints removes them on restore, and the other way round
    g.upload_joints(None)
    bare = g.snapshot()
    g.restore(snap)
    assert len(g.download_joints()) == 50
    g.restore(bare)
    assert len(g.download_joints()) == 0


def test_state_file_round_trip_and_an_older_file(tmp_path):
    s = _pile()
    g, h = nudge_b200.Sim(s), nudge_b200.Sim(s)
    rng = np.random.default_rng(7)
    g.upload_joints(_joints_at_rest(s.transforms, rng, 50, s.n_bodies))
    for _ in range(5):
        g.step()
    old, new = str(tmp_path / "old.nbstate"), str(tmp_path / "new.nbstate")
    h.save_state(old)
    g.save_state(new)
    head = STATE_HEADER.unpack(open(new, "rb").read(STATE_HEADER.size))
    assert head[1] == 6 and head[8 + 6] == 50
    assert STATE_HEADER.unpack(open(old, "rb").read(STATE_HEADER.size))[1] == 1
    h.load_state(new)
    assert h.download_joints().tobytes() == g.download_joints().tobytes()
    for _ in range(5):
        g.step(); h.step()
    assert _body_bytes(g) == _body_bytes(h) and h.download_joints().tobytes() == g.download_joints().tobytes()
    g.load_state(old)
    assert len(g.download_joints()) == 0


def test_refusals_change_nothing():
    s = _pile()
    g = nudge_b200.Sim(s)
    rng = np.random.default_rng(9)
    joints = _joints_at_rest(s.transforms, rng, 20, s.n_bodies)
    g.upload_joints(joints)
    kept = g.download_joints().tobytes()

    def bad(**kw):
        j = joints.copy()
        for k, v in kw.items():
            j[k][7] = v
        return j
    cases = [(bad(a=0), "static world"), (bad(a=5, b=5), "same body"), (bad(a=s.n_bodies), "beyond"), (bad(b=s.n_bodies + 3), "beyond"),
             (bad(type=4), "unknown type"), (bad(length=np.nan), "not finite"), (bad(anchor_a=(0.0, np.inf, 0.0)), "not finite"),
             (bad(impulse=(0.0, 0.0, 0.0, 0.0, 0.0, np.nan)), "not finite")]
    for j, what in cases:
        with pytest.raises(nudge_b200.NudgeError, match=what):
            g.upload_joints(j)
        assert g.download_joints().tobytes() == kept
    assert g.lib.nb_upload_joints(g.ctx, None, 3, g.stream) == -3   # NB_ERR_ARGUMENT
    tower = np.repeat(np.array([_at_rest(s.transforms, joints_ref.BALL, 1, 0, rng)]), 4097)   # 4,097 joints on one body: as many levels
    with pytest.raises(nudge_b200.NudgeError, match="4096 levels"):
        g.upload_joints(tower)
    assert g.download_joints().tobytes() == kept
    g.upload_joints(tower[:4096])
    g.upload_joints(joints)
    # the staged path needs the step's time step before the rows are built
    g.collide(); g.read_cached_impulses()
    with pytest.raises(nudge_b200.NudgeError, match="nb_apply_gravity_damping"):
        g.setup_contact_constraints()
    g.apply_gravity_damping(); g.setup_contact_constraints(); g.apply_impulses(2); g.update_cached_impulses(); g.write_cached_impulses(); g.advance()
    # nb_upload_bodies keeps the set while the body count holds; nb_shard_step refuses it
    g.upload_bodies()
    assert len(g.download_joints()) == 20
    b = nudge_b200.Sim(s)
    b.upload_joints(joints)
    b.shard_create(0, 1, None, 1, 1)
    with pytest.raises(nudge_b200.NudgeError, match="joints"):
        b.shard_step("peer")
    b.upload_joints(None)
    b.shard_step("peer")
    g.reload(scenes.demo_scene(100, 100, iterations=6, spread=3.0, height=12.0))
    assert len(g.download_joints()) == 0
