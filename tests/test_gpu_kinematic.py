"""Kinematic bodies on the device (nb_upload_kinematic_bodies, DESIGN.md section 8.8): no set or an empty set is a plain context bit for bit,
launches included; the ground on a kinematic body at rest is the plain context (and, through the restatement, the reference) with body
indices mapped, on the 8,191-box and the 65,536-box pile; moving platforms (elevator, slider, turntable) equal the restatement
(tests/kinematic_ref.py) at every stage; sleep on a stopped platform and wake when it moves; throughput mode; sensors and contact events on a
kinematic body; graph replay with new velocities every step; state files with nb_replay; and the argument errors."""
import ctypes, os, struct, subprocess, tempfile
import numpy as np
import pytest
import nudge_b200
from nudge_b200 import scenes
from tests.kinematic_ref import KinematicOracleSim, with_kinematic_ground, two_kinematic_platforms
from tests.parity_util import Report, compare_oracle_gpu_step
from tests.gpu_util import fnv1a, side_stream

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NB_ERR_ARGUMENT = -3


def _rows(k, v=(0.0, 0.0, 0.0), w=(0.0, 0.0, 0.0)):
    return np.array([(k, v, w, 0)], scenes.KINEMATIC)


def _state(x):
    x.download_bodies(); x.download_contacts(); x.download_cache()
    c = x.contacts_view()
    parts = [x.transforms, x.momentum, x.idle, c["data"], c["bodies"], c["tags"], c["features"], c["sleeping"], c["active"]]
    cv = x.cache_view()
    return b"".join(np.ascontiguousarray(a).tobytes() for a in parts + [cv["tags"], cv["features"], cv["data"]])


def _mapped_state(x, k):
    """_state of the kinematic-ground context in the plain scene's indices: rows [K, 1..K-1], contact bodies K -> 0."""
    x.download_bodies(); x.download_contacts(); x.download_cache()
    rows = np.array([k] + list(range(1, k)), np.int64)
    c = x.contacts_view()
    b = c["bodies"].copy()
    for f in ("a", "b"):
        b[f][b[f] == k] = 0
    parts = [x.transforms[rows], x.momentum[rows], x.idle[rows], c["data"], b, c["tags"], c["features"], c["sleeping"], c["active"]]
    cv = x.cache_view()
    return b"".join(np.ascontiguousarray(a).tobytes() for a in parts + [cv["tags"], cv["features"], cv["data"]])


def test_no_set_and_empty_set_are_a_plain_context_with_the_same_launches():
    s = scenes.demo_scene(300, 300, iterations=4, spread=8.0, height=14.0, seed=31)
    plain, empty, removed = (nudge_b200.Sim(s, stream=side_stream(), pair_capacity=1 << 16, contact_capacity=1 << 17) for _ in range(3))
    empty.upload_kinematic_bodies(np.zeros(0, scenes.KINEMATIC))
    removed.upload_kinematic_bodies(_rows(5, (0.0, 1.0, 0.0)))
    removed.upload_kinematic_bodies(None)
    removed.download_bodies(); removed.momentum[5] = plain.momentum[5]; removed.upload_bodies()   # the set's removal keeps the written row
    for i in range(60):
        used = []
        for x in (plain, empty, removed):
            before = x.launch_count()
            x.step() if i % 3 else x.step_staged()
            used.append(x.launch_count() - before)
        assert used[0] == used[1] == used[2], (i, used)
        if i % 3:
            assert used[0] == 61, used
        ref = _state(plain)
        assert _state(empty) == ref and _state(removed) == ref, i
        cp, ce = plain.counts(), empty.counts()
        assert (cp.pairs, cp.contacts, cp.batches, cp.active) == (ce.pairs, ce.contacts, ce.batches, ce.active)


@pytest.mark.parametrize("n", [8191, 65536])
def test_kinematic_ground_at_rest_is_the_plain_context_mapped(n):
    base = scenes.box_drop(n, iterations=8)
    ks, k = with_kinematic_ground(base)
    plain, kin = nudge_b200.Sim(base, stream=side_stream()), nudge_b200.Sim(ks, stream=side_stream())
    for i in range(40 if n == 8191 else 20):
        a, b = plain.launch_count(), kin.launch_count()
        plain.step(); kin.step()
        assert plain.launch_count() - a == kin.launch_count() - b
        assert _mapped_state(kin, k) == _state(plain), i
        cp, ck = plain.counts(), kin.counts()
        assert (cp.pairs, cp.contacts, cp.batches, cp.levels, cp.active, cp.sleeping) == (ck.pairs, ck.contacts, ck.batches, ck.levels, ck.active, ck.sleeping), i


def test_kinematic_ground_at_rest_equals_the_restatement_at_every_stage():
    """The restatement reproduces the reference's recorded digests on this scene (tests/test_kinematic_oracle.py)."""
    ks, k = with_kinematic_ground(scenes.box_drop(1500, iterations=8))
    o = KinematicOracleSim(ks, contact_capacity=1 << 17)
    g = nudge_b200.Sim(ks, contact_capacity=o.cap, debug=True)
    for i in range(12):
        rep = Report("step %d" % i)
        assert compare_oracle_gpu_step(o, g, rep), str(rep)


def _platform_scene(v, w):
    base = scenes.box_drop(600, iterations=8, density_L=14.0, spacing=(2.2, 2.4, 2.2), rotate=True)
    return with_kinematic_ground(base, v, w)


@pytest.mark.parametrize("motion", ["elevator", "slider", "turntable"])
def test_moving_platforms_equal_the_restatement_bit_for_bit(motion):
    v, w = {"elevator": ((0.0, 0.5, 0.0), (0.0, 0.0, 0.0)), "slider": ((0.75, 0.0, 0.25), (0.0, 0.0, 0.0)),
            "turntable": ((0.0, 0.0, 0.0), (0.0, 0.4, 0.0))}[motion]
    ks, k = _platform_scene(v, w)
    o = KinematicOracleSim(ks, contact_capacity=1 << 16)
    g = nudge_b200.Sim(ks, contact_capacity=o.cap, debug=True)
    g.download_bodies()
    row = g.momentum[k].copy()
    assert np.array_equal(row["velocity"], np.float32(v)) and np.array_equal(row["angular_velocity"], np.float32(w))
    for i in range(50):
        rep = Report("%s step %d" % (motion, i))
        assert compare_oracle_gpu_step(o, g, rep), str(rep)
        assert g.momentum[k].tobytes() == row.tobytes() or (np.array_equal(g.momentum[k]["velocity"], row["velocity"]) and np.array_equal(g.momentum[k]["angular_velocity"], row["angular_velocity"]))
        assert k in g.contacts_view()["active"].tolist()
    assert g.debug("kind", np.uint8)[k] == 3   # kinematic, moving
    c = g.constraints_view()
    assert (c["a"] >> 31).any() or (c["b"] >> 31).any()   # read-only sides in the rows


def test_pile_sleeps_on_a_stopped_platform_wakes_when_it_moves_and_sleeps_again():
    ks, k = with_kinematic_ground(scenes.box_drop(400, iterations=4, density_L=12.0, spacing=(2.2, 2.2, 2.2), rotate=False))
    g = nudge_b200.Sim(ks, stream=side_stream())

    def until_asleep(limit):
        for i in range(limit):
            g.step()
            if g.counts().active == 0:
                return i
        return None
    assert until_asleep(1500) is not None, "the pile never fell asleep"
    g.upload_kinematic_bodies(_rows(k, (0.0, 0.0, 0.2)))
    g.step()
    g.download_contacts()
    act = g.contacts_view()["active"].tolist()
    assert k in act and len(act) > 300
    for _ in range(60):
        g.step()
    g.download_bodies()
    assert np.array_equal(g.momentum[k]["velocity"], np.float32([0.0, 0.0, 0.2]))
    g.upload_kinematic_bodies(_rows(k))
    assert until_asleep(1500) is not None, "the pile did not fall asleep again"


def test_throughput_mode_leaves_kinematic_rows_alone():
    ks, k = _platform_scene((0.0, 0.3, 0.0), (0.0, 0.2, 0.0))
    g = nudge_b200.Sim(ks)
    g.set_solver_mode("throughput")
    g.download_bodies()
    row = g.momentum[k].copy()
    y0 = float(g.transforms["position"][k, 1])
    for i in range(80):
        g.step()
        g.download_bodies()
        assert g.momentum[k]["velocity"].tobytes() == row["velocity"].tobytes()
        assert g.momentum[k]["angular_velocity"].tobytes() == row["angular_velocity"].tobytes()
    c = g.counts()
    assert c.contacts > 0 and c.overflow == 0 and np.isfinite(g.transforms["position"]).all()
    assert float(g.transforms["position"][k, 1]) > y0 and g.debug("body_contacts", np.uint32)[k] == 0   # never mass-split
    # the boxes above the platform stay above it
    assert (g.transforms["position"][1:k, 1] > g.transforms["position"][k, 1] - 1.0).all()


def test_sensor_contacts_and_pairs_of_a_kinematic_body():
    """A kinematic paddle (box) above the ground with a sensor sphere on it: the sensor overlaps the ground, the paddle's contacts with boxes
    give ordinary events, and no paddle-ground pair reaches the broadphase list."""
    s = scenes.demo_scene(40, 0, iterations=4, spread=1.5, height=3.0, seed=5)
    s.transforms["position"][1:, 1] -= 8.5   # just above the paddle
    k = s.n_bodies
    s.transforms = np.concatenate([s.transforms, s.transforms[:1]]); s.transforms["position"][k] = (0.0, -9.6, 0.0)
    s.properties = np.concatenate([s.properties, s.properties[1:2]])
    s.momentum = np.concatenate([s.momentum, s.momentum[:1]]); s.idle = np.concatenate([s.idle, s.idle[:1]])
    paddle = s.n_boxes
    s.box_tags = np.concatenate([s.box_tags, [np.uint32(1000)]]); s.box_data = np.concatenate([s.box_data, s.box_data[1:2]])
    s.box_data["size"][paddle] = (3.0, 0.5, 3.0)
    s.box_transforms = np.concatenate([s.box_transforms, s.box_transforms[:1]]); s.box_transforms["position"][paddle] = 0; s.box_transforms["body"][paddle] = k
    s.sphere_tags = np.array([1001], np.uint32); s.sphere_data = np.zeros(1, scenes.SPHERE); s.sphere_data["radius"] = 0.5
    s.sphere_transforms = np.zeros(1, scenes.TRANSFORM); s.sphere_transforms["rotation"][:, 3] = 1; s.sphere_transforms["body"] = k
    s.sphere_transforms["position"][0] = (0.0, -0.6, 0.0)   # inside the paddle, reaching into the ground
    s.sensors = np.zeros(s.n_colliders, np.uint8); s.sensors[-1] = 1
    s.kinematic = _rows(k, (0.0, 0.05, 0.0))
    g = nudge_b200.Sim(s, debug=True)
    g.enable_contact_events(1 << 14)
    begins = 0
    for i in range(30):
        g.step_staged()
        keys = g.debug("pair_keys", np.uint64)
        kb = int(g.debug_scalar("kbits"))
        lo, hi = keys & np.uint64((1 << kb) - 1), keys >> np.uint64(kb)
        assert not (((lo == 0) & (hi == paddle)) | ((lo == paddle) & (hi == 0))).any(), i   # ground (collider 0) and paddle: never a pair
        ov = g.sensor_overlaps()
        assert (ov["tags"] == np.uint64(1001 << 32)).any(), i    # the sensor sphere on the kinematic body reaches into the ground (tag 0)
        ev, _ = g.contact_events()
        begins += int(((ev["kind"] == scenes.CONTACT_BEGIN) & ((ev["body_a"] == k) | (ev["body_b"] == k))).sum())
    assert begins > 0


def test_graph_replay_with_new_velocities_every_step():
    ks, k = _platform_scene((0.0, 0.0, 0.0), (0.0, 0.0, 0.0))
    a, b = nudge_b200.Sim(ks, stream=side_stream()), nudge_b200.Sim(ks, stream=side_stream())
    plain = ks.copy(); plain.kinematic = None
    c = nudge_b200.Sim(plain, stream=side_stream())
    a.step(); b.step_staged(); c.step()
    before = c.launch_count(); c.step()
    per_step = c.launch_count() - before   # a context without a set
    for i in range(1, 30):
        r = _rows(k, (0.0, 0.02 * i, 0.01), (0.0, 0.01 * i, 0.0))
        before = a.launch_count()
        a.upload_kinematic_bodies(r); b.upload_kinematic_bodies(r)
        a.step(); b.step_staged()
        assert a.launch_count() - before == per_step + 1, i   # the scatter and the replayed step
        assert _state(a) == _state(b), i
    assert a.debug_scalar("graph_active") == 1
    # a changed set re-records: the same result as the stage calls, and the graph stays in use
    r = np.concatenate([_rows(k, (0.0, 0.1, 0.0)), _rows(7, (0.0, 0.0, 0.0))])
    a.upload_kinematic_bodies(r); b.upload_kinematic_bodies(r)
    for i in range(5):
        a.step(); b.step_staged()
        assert _state(a) == _state(b), i
    assert a.debug_scalar("graph_active") == 1


def test_state_files_carry_the_set_and_replay():
    side = side_stream()
    ks, k = _platform_scene((0.0, 0.2, 0.0), (0.0, 0.1, 0.0))
    g = nudge_b200.Sim(ks, stream=side)
    for _ in range(20):
        g.step()
    d = tempfile.mkdtemp(prefix="nb_kinematic_state_")
    p1, p2, p3 = (os.path.join(d, x) for x in ("a.bin", "b.bin", "plain.bin"))
    g.save_state(p1)
    raw = open(p1, "rb").read()
    version, = struct.unpack_from("<I", raw, 8); reserved = struct.unpack_from("<8I", raw, 36)
    assert version == 4 and reserved[4] == 1 and reserved[2] == 0
    assert struct.unpack_from("<I", raw, len(raw) - 16)[0] == k
    h = nudge_b200.Sim(_platform_scene((0.0, 0.0, 0.0), (0.0, 0.0, 0.0))[0], stream=side)
    h.upload_kinematic_bodies(None)
    h.load_state(p1)
    for i in range(10):
        g.step(); h.step()
        assert _state(g) == _state(h), i
    exe = os.path.join(ROOT, "tools", "bin", "nb_replay")
    out = subprocess.run([exe, p1, "--steps", "10", "--iterations", str(int(ks.iterations)), "--dump", p2], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stdout + out.stderr
    last = out.stdout.strip().splitlines()[-1].split()
    h.load_state(p1)
    for _ in range(10):
        h.step()
    h.download_bodies()
    assert int(last[last.index("xf") + 1], 16) == fnv1a(h.transforms.tobytes())
    assert open(p2, "rb").read()[8:12] == struct.pack("<I", 4)
    # a version-1 file drops the set: the platform is dynamic again and falls
    plain = nudge_b200.Sim(with_kinematic_ground(scenes.box_drop(600, iterations=8, density_L=14.0, spacing=(2.2, 2.4, 2.2)))[0], stream=side)
    plain.upload_kinematic_bodies(None)
    plain.save_state(p3)
    assert struct.unpack_from("<I", open(p3, "rb").read(), 8)[0] == 1
    h.load_state(p3)
    h.download_bodies(); y0 = float(h.transforms["position"][k, 1])
    h.step(); h.step()
    h.download_bodies()
    assert float(h.transforms["position"][k, 1]) < y0


def test_argument_errors_shard_refusal_and_body_count_change():
    ks, k = _platform_scene((0.0, 0.1, 0.0), (0.0, 0.0, 0.0))
    g = nudge_b200.Sim(ks)
    g.step_staged()
    for bad in (_rows(0), _rows(ks.n_bodies), np.concatenate([_rows(5), _rows(5)])):
        r = np.ascontiguousarray(bad)
        assert g.lib.nb_upload_kinematic_bodies(g.ctx, r.ctypes.data_as(ctypes.c_void_p), len(r), g.stream) == NB_ERR_ARGUMENT
    g.download_bodies()
    assert g.debug("kind", np.uint8)[k] & 1 and g.momentum[k]["velocity"][1] == np.float32(0.1)   # the set and its rows are unchanged
    b = nudge_b200.Sim(ks)
    b.shard_create(0, 1, None, 1, 1)
    with pytest.raises(nudge_b200.NudgeError, match="kinematic"):
        b.shard_step("peer")
    b.upload_kinematic_bodies(None)
    b.shard_step("peer")
    # nb_upload_bodies with the same count keeps the set, another count drops it
    g.upload_bodies()
    assert len(g.debug("kind", np.uint8)) == ks.n_bodies
    smaller = scenes.box_drop(599, iterations=8, density_L=14.0, spacing=(2.2, 2.4, 2.2))
    g.reload(smaller)
    assert len(g.debug("kind", np.uint8)) == 0
    g.step_staged()


def test_two_kinematic_bodies_collide_equals_the_restatement_every_step():
    """Two kinematic slabs overlapping each other and the ground on body 0 (tests/kinematic_ref.two_kinematic_platforms): the device steps, and
    every step its collide stage (pairs, contacts, active bodies, sleeping pairs) equals the restatement's from the same state, while K1
    rises, K2 stops and starts, and the pile is put to sleep."""
    from tests.parity_util import sync_oracle_from_gpu
    s, k1, k2 = two_kinematic_platforms()
    o = KinematicOracleSim(s, contact_capacity=1 << 16)
    g = nudge_b200.Sim(s, contact_capacity=o.cap, debug=True)
    rows = lambda v1, v2: np.array([(k1, v1, (0.0, 0.0, 0.0), 0), (k2, v2, (0.0, 0.0, 0.0), 0)], scenes.KINEMATIC)
    sleeping = 0
    for i in range(80):
        if i in (0, 30, 50):
            r = {0: rows((0.0, 0.1, 0.0), (0.0, 0.0, 0.0)), 30: rows((0.0, 0.0, 0.0), (0.0, 0.0, 0.0)), 50: rows((0.0, 0.0, 0.0), (0.2, 0.0, 0.0))}[i]
            g.upload_kinematic_bodies(r)
        if i in (25, 45):   # the whole pile asleep and at rest
            g.download_bodies(); g.idle[1:k1] = 0xff; g.momentum["velocity"][1:k1] = 0; g.momentum["angular_velocity"][1:k1] = 0; g.upload_bodies()
        sync_oracle_from_gpu(o, g)
        o.collide(); g.collide(); g.download_contacts()
        rep = Report("step %d" % i)
        op, gp = o.pairs_view(), g.pairs_view()
        rep.eq("pairs.lo", op["lo"], gp["lo"]); rep.eq("pairs.hi", op["hi"], gp["hi"])
        oc, gc = o.contacts_view(), g.contacts_view()
        for f in ("data", "bodies", "tags", "features", "sleeping", "active"):
            rep.eq(f, oc[f], gc[f])
        assert rep.ok, str(rep)
        sleeping += len(gc["sleeping"])
        g.apply_gravity_damping(); g.read_cached_impulses(); g.setup_contact_constraints(); g.apply_impulses(int(s.iterations))
        g.update_cached_impulses(); g.write_cached_impulses(); g.advance()
    g.download_bodies()
    assert np.array_equal(g.momentum["velocity"][k2], np.float32([0.2, 0.0, 0.0])) and sleeping > 0


def test_ball_joint_chain_hung_from_a_moving_kinematic_body_follows_it():
    """A 6-link chain of ball joints (tests/test_gpu_rows.ball_joint_rows) hung from a kinematic hook that moves sideways: the user rows
    treat the hook as infinite mass and never write it (its momentum row stays byte-identical every step), the joint error stays bounded
    and the chain follows the hook."""
    from tests.test_gpu_rows import ball_joint_rows, _quat_rotate
    links = 6
    s = scenes.demo_scene(links + 1, 0, iterations=12, spread=3.0, height=6.0, seed=5)
    hook = links + 1
    s.box_data["size"][1:links + 1] = (0.2, 0.5, 0.2)
    s.properties[1:links + 1] = scenes._box_props(s.box_data["size"][1:links + 1])
    s.box_data["size"][hook] = (0.2, 0.2, 0.2)
    top = np.array([0.0, 8.0, 0.0])
    s.transforms["position"][hook] = top; s.transforms["rotation"][hook] = (0.0, 0.0, 0.0, 1.0)
    for k in range(links):                                    # hanging straight down from the hook
        s.transforms["position"][1 + k] = top - np.array([0.0, 0.75 + 1.0 * k, 0.0])
        s.transforms["rotation"][1 + k] = (0.0, 0.0, 0.0, 1.0)
    s.connections = np.zeros(links, scenes.PAIR32)
    s.connections["a"] = np.arange(1, links + 1); s.connections["b"] = np.concatenate([[hook], np.arange(1, links)])
    v = np.float32([0.6, 0.0, 0.0])
    s.kinematic = _rows(hook, tuple(v))
    g = nudge_b200.Sim(s)
    g.download_bodies()
    row = g.momentum[hook].tobytes()
    x0 = g.transforms["position"][hook].copy()
    dt = float(s.time_step)
    worst = 0.0
    for step in range(240):
        g.download_bodies()
        rows = [ball_joint_rows(g.transforms, 1, hook, (0.0, 0.5, 0.0), (0.0, -0.25, 0.0), dt)]
        for k in range(1, links):
            rows.append(ball_joint_rows(g.transforms, 1 + k, k, (0.0, 0.5, 0.0), (0.0, -0.5, 0.0), dt))
        g.upload_constraint_rows(np.concatenate(rows))
        g.step_staged()
        g.download_bodies()
        assert g.momentum[hook].tobytes() == row, step
        if step > 20:
            xf = g.transforms
            wa = xf["position"][1] + _quat_rotate(xf["rotation"][1].astype(np.float64), np.array([0.0, 0.5, 0.0]))
            worst = max(worst, float(np.linalg.norm(wa - (xf["position"][hook] + np.array([0.0, -0.25, 0.0])))))
            for k in range(1, links):
                wa = xf["position"][1 + k] + _quat_rotate(xf["rotation"][1 + k].astype(np.float64), np.array([0.0, 0.5, 0.0]))
                wb = xf["position"][k] + _quat_rotate(xf["rotation"][k].astype(np.float64), np.array([0.0, -0.5, 0.0]))
                worst = max(worst, float(np.linalg.norm(wa - wb)))
    moved = g.transforms["position"][hook] - x0
    assert abs(float(moved[0]) - 240 * dt * 0.6) < 1e-3 and moved[1] == 0.0
    assert worst < 0.08, worst
    assert abs(float(g.transforms["position"][1, 0] - g.transforms["position"][hook, 0])) < 0.6     # the top link hangs from the hook
    assert float(g.transforms["position"][links, 0] - x0[0]) > 0.25 * float(moved[0])              # the end has been dragged along
    assert np.isfinite(g.transforms["position"]).all() and g.counts().overflow == 0


def test_state_versions_3_and_4_with_sensors():
    """Sensors and a set: version 4 with reserved[2] = 1 carries both; loading a version-3 file (sensors, no set) removes a set."""
    from tests.sensor_ref import add_sensors
    side = side_stream()
    ks, k = _platform_scene((0.0, 0.2, 0.0), (0.0, 0.0, 0.0))
    kin = ks.kinematic
    ks = add_sensors(ks, zones=[((0.0, 1.0, 0.0), (3.0, 1.0, 3.0))])
    ks.kinematic = kin
    g = nudge_b200.Sim(ks, stream=side)
    for _ in range(30):
        g.step()
    d = tempfile.mkdtemp(prefix="nb_kinematic_state_")
    p4, p3 = os.path.join(d, "v4.bin"), os.path.join(d, "v3.bin")
    g.save_state(p4)
    raw = open(p4, "rb").read()
    version, = struct.unpack_from("<I", raw, 8); reserved = struct.unpack_from("<8I", raw, 36)
    assert version == 4 and reserved[2] == 1 and reserved[4] == 1
    other = ks.copy(); other.kinematic = None; other.sensors = None
    h = nudge_b200.Sim(other, stream=side)
    h.load_state(p4)
    assert h.debug("kind", np.uint8)[k] & 1
    for i in range(10):
        g.step(); h.step()
        assert _state(g) == _state(h) and g.sensor_overlaps().tobytes() == h.sensor_overlaps().tobytes(), i
    assert len(g.sensor_overlaps()) > 0
    g.upload_kinematic_bodies(None)   # the rows stay as they are: stop the platform, so that as a dynamic body it can only fall
    g.download_bodies(); g.momentum["velocity"][k] = 0; g.momentum["angular_velocity"][k] = 0; g.upload_bodies()
    g.save_state(p3)
    assert struct.unpack_from("<I", open(p3, "rb").read(), 8)[0] == 3
    assert len(h.debug("kind", np.uint8)) == ks.n_bodies
    h.load_state(p3)
    assert len(h.debug("kind", np.uint8)) == 0
    h.download_bodies(); y0 = float(h.transforms["position"][k, 1])
    h.step(); h.step()
    h.download_bodies()
    assert float(h.transforms["position"][k, 1]) < y0     # dynamic again: it falls
