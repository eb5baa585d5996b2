"""Continuous collision (nb_upload_ccd_bodies; DESIGN.md section 8.18) on the device.

- Without a set, with an empty set and with a set whose thresholds are all +inf, 100 graph-replayed steps are byte for byte a plain
  context's, with its launch count (one more, k_ccd, for the +inf set).
- Per step against the numpy restatement (oracle/ccd_ref.py) on a settled 8k-box pile with about 1,000 listed bodies, a quarter of them
  fired into it, and on a mixed box / ball scene over a static ground, in both solver modes: every listed body's (t, collider), read back
  through nb_debug_read("ccd_hits"), is ccd_ref's, and every advanced body's position is p + (v * dt) * t in float32 (t = 1 off the set),
  with p before the step and v the step's velocities.  In parity mode also, before each step, a twin loads the context's state file and
  removes its set, and after the step every byte equals the twin's except the positions of clamped bodies.  (Throughput mode sums velocity
  changes with float reductions in no fixed order, so two contexts need not agree bit for bit there, with or without a set.)
- nb_step's graph replay against the staged calls, with one graph record.
- Tunnelling: 256 small boxes fired at 120 m/s through a 0.2-thick static wall pass it without a set and stop on its near side with one;
  boxes dropped from 500 m onto a thin static plate fall through it without a set and rest on it with one.
- Bodies clamped against a wall of non-round extents and turned away from it or along its face move on the next step; a listed body
  made kinematic is never clamped.
- Re-uploads that keep or re-record the graph, nb_remove_bodies renumbering, nb_add_bodies, snapshot restores re-stepped bit for bit, a
  version-8 state file through nb_load_state and tools/nb_replay, a context without a set writing the bytes it wrote before, every
  refusal changing nothing, nb_shard_step refused.
- In-scene casts on the mixed scene and on a level-8 scene record no grid fallbacks."""
import ctypes, os, struct, subprocess, tempfile
import numpy as np
import pytest
import nudge_b200
from nudge_b200 import abi, scenes
from oracle import ccd_ref, raycast_ref
from tests.gpu_util import fnv1a, side_stream
from tests.test_gpu_raycast import small_mixed_scene

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NB_ERR_ARGUMENT = -3
INF = float("inf")


def _rows(bodies, radius=0.3, threshold=0.0, category=0xffff, mask=0xffff):
    e = np.zeros(len(bodies), abi.CCD_BODY)
    e["body"], e["radius"], e["motion_threshold"], e["category"], e["mask"] = bodies, radius, threshold, category, mask
    return e


def _state(x, positions=True):
    """The bytes a step leaves: bodies (positions optional), contacts, active list and cache."""
    x.download_bodies(); x.download_contacts(); x.download_cache()
    c, cv = x.contacts_view(), x.cache_view()
    xf = [x.transforms] if positions else [x.transforms["rotation"], x.transforms["body"]]
    parts = xf + [x.momentum, x.idle, c["data"], c["bodies"], c["tags"], c["features"], c["sleeping"], c["active"],
             cv["tags"], cv["features"], cv["data"]]
    return b"".join(np.ascontiguousarray(a).tobytes() for a in parts)


def _settled(scene, steps, mode="parity"):
    sim = nudge_b200.Sim(scene, stream=side_stream())
    sim.set_solver_mode(mode)
    for _ in range(steps):
        sim.step()
    return sim


@pytest.fixture(scope="module")
def pile8k():
    return scenes.box_drop(8192, seed=4), 300


@pytest.fixture(scope="module")
def mixed():
    return scenes.demo_scene(2000, 2000, iterations=8, spread=12.0, height=30.0, seed=6), 200


def test_no_set_empty_set_and_infinite_thresholds_are_a_plain_context():
    s = scenes.demo_scene(300, 300, iterations=4, spread=8.0, height=14.0, seed=31)
    plain, empty, never = (nudge_b200.Sim(s, stream=side_stream(), pair_capacity=1 << 16, contact_capacity=1 << 17) for _ in range(3))
    empty.upload_ccd_bodies(np.zeros(0, abi.CCD_BODY))
    never.upload_ccd_bodies(_rows(np.arange(1, s.n_bodies), 0.2, INF))
    for i in range(100):
        used = []
        for x in (plain, empty, never):
            before = x.launch_count()
            x.step()
            used.append(x.launch_count() - before)
        assert used == [61, 61, 62], (i, used)
        ref = _state(plain)
        assert _state(empty) == ref and _state(never) == ref, i
    assert never.debug("ccd_hits", np.uint32).reshape(-1, 2).tolist() == [[0x3f800000, abi.RAY_NO_HIT]] * (s.n_bodies - 1)
    assert plain.debug_scalar("graph_records") == empty.debug_scalar("graph_records") == never.debug_scalar("graph_records") == 1


def _fire(sim, bodies, rng, speed):
    """Sets the listed bodies' velocities to `speed` in random directions (downwards-leaning, into the pile)."""
    sim.download_bodies()
    v = rng.normal(size=(len(bodies), 3)); v[:, 1] = -np.abs(v[:, 1]) - 0.5
    sim.momentum["velocity"][bodies] = speed * v / np.linalg.norm(v, axis=1, keepdims=True)
    sim.upload_bodies()


def _check_steps(sim, twin, entries, steps, path, staged_every=0):
    """Steps sim (with its set) `steps` times against the restatement and, with a twin (parity mode), against the twin without the set loaded
    from sim's state before each step.  Returns the number of clamped entries over the steps."""
    s = sim.scene
    dt = np.float32(s.time_step)
    bodies = entries["body"].astype(np.int64)
    clamped = 0
    for i in range(steps):
        if twin is not None:
            sim.save_state(path)
            twin.load_state(path)
            twin.upload_ccd_bodies(None)
        sim.download_bodies()
        p0 = sim.transforms["position"].copy()
        scene = raycast_ref.Scene.of_sim(sim, s.collision_filters, s.sensors)
        staged = staged_every and i % staged_every == 0
        for x in (sim, twin) if twin is not None else (sim,):
            (x.step_staged if staged else x.step)()
        if twin is not None:
            assert _state(sim, positions=False) == _state(twin, positions=False), i
        else:
            _state(sim)
        active = np.zeros(s.n_bodies, bool); active[sim.contacts_view()["active"].astype(np.int64)] = True
        active[0] = False
        t, col, pos = ccd_ref.step(scene, entries, p0[bodies], sim.momentum["velocity"][bodies], dt, active[bodies])
        hits = sim.debug("ccd_hits", np.uint32).reshape(-1, 2)
        assert (hits[:, 0] == t.view(np.uint32)).all() and (hits[:, 1] == col).all(), (i, np.nonzero((hits[:, 1] != col))[0][:5])
        got = sim.transforms["position"]
        assert got[bodies].tobytes() == pos.tobytes(), i
        factor = np.ones(s.n_bodies, np.float32); factor[bodies] = t   # every advanced body: p + (v * dt) * t, the others stay
        want = np.where(active[:, None], p0 + (sim.momentum["velocity"] * dt) * factor[:, None], p0)
        assert got.tobytes() == want.astype(np.float32).tobytes(), i
        hit = col != ccd_ref.NO_HIT
        if twin is not None:
            keep = np.ones(s.n_bodies, bool); keep[bodies[hit]] = False
            assert got[keep].tobytes() == twin.transforms["position"][keep].tobytes(), i
        clamped += int(hit.sum())
    return clamped


@pytest.mark.parametrize("mode", ["parity", "throughput"])
def test_settled_pile_with_fast_bodies_equals_the_restatement_every_step(pile8k, mode, tmp_path):
    scene, settle = pile8k
    sim = _settled(scene, settle, mode)
    twin = nudge_b200.Sim(scene, stream=side_stream()) if mode == "parity" else None
    rng = np.random.default_rng(11)
    bodies = np.sort(rng.choice(np.arange(1, scene.n_bodies), 1000, replace=False)).astype(np.uint32)
    entries = _rows(bodies, rng.uniform(0.05, 0.45, 1000).astype(np.float32), np.where(np.arange(1000) % 4 == 0, 0.05, 0.0).astype(np.float32))
    entries["motion_threshold"][::97] = INF
    sim.upload_ccd_bodies(entries)
    _fire(sim, bodies[::4], rng, 90.0)
    assert _check_steps(sim, twin, entries, 60, str(tmp_path / "s.bin"), staged_every=7) >= 10
    assert sim.debug_scalar("ccd_fallbacks") == 0


@pytest.mark.parametrize("mode", ["parity", "throughput"])
def test_mixed_scene_fast_balls_and_boxes_over_static_ground_equal_the_restatement(mixed, mode, tmp_path):
    scene, settle = mixed
    sim = _settled(scene, settle, mode)
    twin = nudge_b200.Sim(scene, stream=side_stream()) if mode == "parity" else None
    rng = np.random.default_rng(12)
    bodies = np.sort(rng.choice(np.arange(1, scene.n_bodies), 800, replace=False)).astype(np.uint32)
    sim.upload_ccd_bodies(_rows(bodies, 0.2))
    _fire(sim, bodies[::2], rng, 90.0)
    assert _check_steps(sim, twin, _rows(bodies, 0.2), 60, str(tmp_path / "s.bin"), staged_every=5) >= 40
    assert sim.debug_scalar("ccd_fallbacks") == 0


def test_graph_replay_equals_the_staged_calls_with_one_record(mixed):
    scene, settle = mixed
    a, b = _settled(scene, settle), _settled(scene, settle)
    bodies = np.arange(1, scene.n_bodies, 5, dtype=np.uint32)
    for x in (a, b):
        x.upload_ccd_bodies(_rows(bodies, 0.25))
        _fire(x, bodies[::3], np.random.default_rng(5), 80.0)
    records = a.debug_scalar("graph_records")
    for i in range(40):
        a.step(); b.step_staged()
        assert _state(a) == _state(b), i
        assert a.debug("ccd_hits", np.uint32).tobytes() == b.debug("ccd_hits", np.uint32).tobytes(), i
    assert a.debug_scalar("graph_records") == records + 1


def _wall_scene(rows=4, cols=64, speed=120.0, wall=True):
    """rows x cols boxes of half extent 0.1 at x = -10.9, just above the standard ground (top at y = -10), moving at `speed` along +x,
    dt = 1/60; a static wall of half thickness 0.1 at x = 0 on body 0."""
    k = rows * cols
    y, z = np.meshgrid(-9.85 + 0.25 * np.arange(rows), -9.6 + 0.3 * np.arange(cols), indexing="ij")
    pos = np.stack([np.full(k, -10.9), y.ravel(), z.ravel()], 1).astype(np.float32)
    s = scenes._assemble("bullets", np.full((k, 3), 0.1, np.float32), pos, None, np.zeros(0, np.float32), np.zeros((0, 3), np.float32))
    if wall:
        s.box_tags = np.append(s.box_tags, np.uint32(s.n_boxes))
        wd = np.zeros(1, scenes.BOX); wd["size"] = (0.1, 20.0, 20.0)
        wt = np.zeros(1, scenes.TRANSFORM); wt["rotation"][0, 3] = 1.0; wt["position"] = (0.0, -10.0, 0.0)
        s.box_data = np.concatenate([s.box_data, wd]); s.box_transforms = np.concatenate([s.box_transforms, wt])
        s.sphere_tags = s.sphere_tags + np.uint32(1)
    s.momentum["velocity"][1:] = (speed, 0.0, 0.0)
    s.time_step = np.float32(1.0 / 60.0)
    return s


def test_bullets_tunnel_through_a_thin_wall_without_the_set_and_stop_with_it():
    s = _wall_scene()
    k = s.n_bodies - 1
    plain = nudge_b200.Sim(s, stream=side_stream())
    ccd = nudge_b200.Sim(s, stream=side_stream())
    ccd.upload_ccd_bodies(_rows(np.arange(1, k + 1), 0.09))
    for i in range(120):
        plain.step(); ccd.step()
        ccd.download_bodies()
        assert (ccd.transforms["position"][1:, 0] < 0.1).all(), i   # no centre ever crosses the far face
    plain.download_bodies()
    assert (plain.transforms["position"][1:, 0] > 0.1).all()      # the scene tunnels
    x, v = ccd.transforms["position"][1:, 0], ccd.momentum["velocity"][1:]
    assert (x < -0.1).all() and (np.linalg.norm(v, axis=1) < 0.5).all(), (x.max(), np.abs(v).max())
    assert ccd.debug_scalar("ccd_fallbacks") == 0


def test_bodies_clamped_against_a_wall_of_any_extent_move_away_and_along_it(tmp_path):
    """256 boxes of random, non-round half extents (spheres at 0.95 of the smallest) fired at a wall of non-round half thickness.  Right
    after its clamp each body is turned away from the wall or along its face; the next step must move it (no t = 0 hit on the wall, where
    the face slab may count the clamped start as inside while step 0 does not), exactly as the restatement says."""
    rng = np.random.default_rng(23)
    n = 256
    sizes = rng.uniform(0.1, 0.3, (n, 3)).astype(np.float32)
    y, z = np.meshgrid(-7.5 + np.arange(16), -7.5 + np.arange(16), indexing="ij")
    pos = np.stack([rng.uniform(-12.5, -11.5, n), y.ravel(), z.ravel()], 1).astype(np.float32)
    s = scenes._assemble("walls", sizes, pos, None, np.zeros(0, np.float32), np.zeros((0, 3), np.float32))
    s.box_tags = np.append(s.box_tags, np.uint32(s.n_boxes))
    wd = np.zeros(1, scenes.BOX); wd["size"] = (0.33663276, 20.0, 20.0)
    wt = np.zeros(1, scenes.TRANSFORM); wt["rotation"][0, 3] = 1.0
    s.box_data = np.concatenate([s.box_data, wd]); s.box_transforms = np.concatenate([s.box_transforms, wt])
    s.momentum["velocity"][1:] = (120.0, 0.0, 0.0)
    s.time_step, s.gravity = np.float32(1.0 / 60.0), np.float32(0.0)
    wall = s.n_boxes - 1
    sim = nudge_b200.Sim(s, stream=side_stream())
    entries = _rows(np.arange(1, n + 1), 0.95 * sizes.min(axis=1))
    sim.upload_ccd_bodies(entries)
    turns = np.array([(-5.0, 0.0, 0.0), (0.0, 5.0, 0.0), (0.0, 0.0, -5.0)], np.float32)   # away, along y, along z
    turned, last = np.zeros(n, bool), np.zeros(n, bool)
    for i in range(12):
        sim.download_bodies()
        p0 = sim.transforms["position"][1:].copy()
        _check_steps(sim, None, entries, 1, str(tmp_path / "s.bin"))
        hits = sim.debug("ccd_hits", np.uint32).reshape(-1, 2)
        assert (hits[last, 1] != wall).all(), (i, np.nonzero(last & (hits[:, 1] == wall))[0][:5])
        assert (sim.transforms["position"][1:][last] != p0[last]).any(axis=1).all(), i
        new = (hits[:, 1] == wall) & ~turned
        if new.any():
            k = np.nonzero(new)[0]
            sim.momentum["velocity"][k + 1] = turns[k % 3]; sim.momentum["angular_velocity"][k + 1] = 0.0
            sim.upload_bodies()
        last, turned = new, turned | new
    sim.download_bodies()
    # a body whose discrete step already lands it overlapping the wall (a start) gets an ordinary contact instead of a clamp
    assert turned.sum() >= 200 and (sim.transforms["position"][1:, 0] < 0.33663276).all(), turned.sum()


def test_a_listed_body_made_kinematic_is_not_clamped():
    s = _wall_scene(rows=1, cols=4)
    sim = nudge_b200.Sim(s, stream=side_stream())
    sim.upload_ccd_bodies(_rows(np.arange(1, 5), 0.09))
    sim.upload_kinematic_bodies(np.array([(1, (120.0, 0.0, 0.0), (0.0, 0.0, 0.0), 0)], scenes.KINEMATIC))
    for i in range(12):
        sim.step()
        assert sim.debug("ccd_hits", np.uint32).reshape(-1, 2)[0].tolist() == [0x3f800000, abi.RAY_NO_HIT], i
    sim.download_bodies()
    x = sim.transforms["position"][1:5, 0]
    assert x[0] > 0.1 and (x[1:] < -0.1).all(), x   # the kinematic body passes the wall, the dynamic ones stop before it
    assert sim.download_ccd_bodies()["body"].tolist() == [1, 2, 3, 4]


def test_a_box_dropped_from_500_m_rests_on_a_thin_plate():
    n = 8
    pos = np.stack([np.arange(n) * 1.5 - 5.0, 500.0 + 0.21 * np.arange(n), np.zeros(n)], 1).astype(np.float32)
    s = scenes._assemble("drop", np.full((n, 3), 0.25, np.float32), pos, None, np.zeros(0, np.float32), np.zeros((0, 3), np.float32),
                         ground_half=(10.0, 0.02, 10.0), ground_y=0.0)
    s.time_step = np.float32(1.0 / 60.0)
    s.damping = np.float32(0.0)   # about 99 m/s at the plate: 1.65 m a step against 0.54 m of box and plate
    plain, ccd = nudge_b200.Sim(s, stream=side_stream()), nudge_b200.Sim(s, stream=side_stream())
    ccd.upload_ccd_bodies(_rows(np.arange(1, n + 1), 0.24))
    for i in range(900):
        plain.step(); ccd.step()
        if i % 10 == 9:
            ccd.download_bodies()
            assert (ccd.transforms["position"][1:, 1] > 0.0).all(), i
    plain.download_bodies()
    assert (plain.transforms["position"][1:, 1] < -0.02).any()   # without the set boxes fall through the plate
    ccd.download_bodies()
    y, v = ccd.transforms["position"][1:, 1], ccd.momentum["velocity"][1:]
    assert (y > 0.02).all() and (y < 0.4).all() and (np.linalg.norm(v, axis=1) < 0.5).all(), (y, v)


def test_reuploads_keep_or_rerecord_the_graph(mixed):
    scene, settle = mixed
    g = _settled(scene, 5)
    bodies = np.arange(1, 200, dtype=np.uint32)
    g.upload_ccd_bodies(_rows(bodies, 0.2)); g.step()
    r = g.debug_scalar("graph_records")
    for rad, thr in ((0.1, 0.0), (0.3, 1.0), (0.0, INF)):   # new radii, thresholds and filters for the same bodies: the same graph
        e = _rows(bodies[::-1], rad, thr, category=0x0003, mask=0x00ff)
        g.upload_ccd_bodies(e); g.step()
        assert g.debug_scalar("graph_records") == r
        assert g.download_ccd_bodies().tobytes() == e[::-1].tobytes()
    g.upload_ccd_bodies(_rows(bodies[1:], 0.2)); g.step()   # another body list: one record
    assert g.debug_scalar("graph_records") == r + 1
    g.upload_ccd_bodies(None); g.step()
    assert g.debug_scalar("graph_records") == r + 2 and len(g.download_ccd_bodies()) == 0


def test_remove_and_add_bodies_and_body_count_changes(mixed):
    scene, settle = mixed
    g = _settled(scene, 5)
    g.upload_ccd_bodies(_rows([5, 10, 20, 40], 0.2))
    g.remove_bodies([7, 10])
    assert g.download_ccd_bodies()["body"].tolist() == [5, 18, 38]
    g.step()
    n = g.scene.n_bodies
    g.add_bodies(scenes.fragment(np.array([[0.0, 40.0, 0.0], [3.0, 40.0, 0.0]], np.float32), first_tag=1 << 20))
    assert g.download_ccd_bodies()["body"].tolist() == [5, 18, 38] and g.scene.n_bodies == n + 2
    g.step()
    g.upload_bodies()   # the same count keeps the set
    assert len(g.download_ccd_bodies()) == 3
    g.reload(scenes.demo_scene(100, 100, iterations=4, seed=3))   # another count removes it
    assert len(g.download_ccd_bodies()) == 0
    g.step()


def test_snapshot_restore_restepped_bit_for_bit(mixed):
    scene, settle = mixed
    g = _settled(scene, settle)
    bodies = np.arange(1, scene.n_bodies, 3, dtype=np.uint32)
    g.upload_ccd_bodies(_rows(bodies, 0.2))
    _fire(g, bodies[::5], np.random.default_rng(9), 70.0)
    snap = g.snapshot()
    run = []
    for _ in range(15):
        g.step(); run.append((_state(g), g.debug("ccd_hits", np.uint32).tobytes()))
    g.upload_ccd_bodies(_rows(bodies[:10], 0.1))   # a different set, then back to the snapshot's
    g.restore(snap)
    assert g.download_ccd_bodies().tobytes() == _rows(bodies, 0.2).tobytes()
    for i in range(15):
        g.step()
        assert (_state(g), g.debug("ccd_hits", np.uint32).tobytes()) == run[i], i


def test_state_file_version_8_round_trip_and_replay(mixed):
    scene, settle = mixed
    side = side_stream()
    g = _settled(scene, 20)
    d = tempfile.mkdtemp(prefix="nb_ccd_state_")
    p0, p1, p2, p3 = (os.path.join(d, x) for x in ("before.bin", "a.bin", "replayed.bin", "after.bin"))
    g.save_state(p0)
    bodies = np.arange(1, scene.n_bodies, 7, dtype=np.uint32)
    e = _rows(bodies, 0.2, 0.01, category=0x0001, mask=0xfffe)
    g.upload_ccd_bodies(e)
    _fire(g, bodies[::5], np.random.default_rng(3), 70.0)
    g.save_state(p1)
    raw = open(p1, "rb").read()
    assert struct.unpack_from("<I", raw, 8)[0] == 8 and struct.unpack_from("<4I", raw, 68) == (len(bodies), 0, 0, 0)
    assert raw[len(raw) - 16 * len(bodies):] == e.tobytes()
    h = nudge_b200.Sim(scene, stream=side)
    h.load_state(p1)
    assert h.download_ccd_bodies().tobytes() == e.tobytes()
    g.save_state(p3)
    for i in range(10):
        g.step(); h.step()
        assert _state(g) == _state(h), i
    exe = os.path.join(ROOT, "tools", "bin", "nb_replay")
    out = subprocess.run([exe, p3, "--steps", "10", "--iterations", str(int(scene.iterations)), "--dump", p2], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stdout + out.stderr
    last = out.stdout.strip().splitlines()[-1].split()
    g.download_bodies()
    assert int(last[last.index("xf") + 1], 16) == fnv1a(g.transforms.tobytes())
    assert open(p2, "rb").read()[8:12] == struct.pack("<I", 8)
    # without a set a context writes what it wrote before: the version and bytes of a save before any set, and an older file removes the set
    h.load_state(p0)
    assert len(h.download_ccd_bodies()) == 0
    h.save_state(p3)
    assert open(p3, "rb").read() == open(p0, "rb").read() and struct.unpack_from("<I", open(p0, "rb").read(), 8)[0] < 8


def test_refusals_change_nothing():
    s = scenes.demo_scene(100, 100, iterations=4, seed=8)
    g = nudge_b200.Sim(s, stream=side_stream())
    g.upload_kinematic_bodies(np.array([(9, (0.0, 0.0, 0.0), (0.0, 0.0, 0.0), 0)], scenes.KINEMATIC))
    good = _rows([3, 4], 0.2)
    g.upload_ccd_bodies(good)
    g.step()
    before = _state(g)
    nan = float("nan")
    for bad in (_rows([0]), _rows([s.n_bodies]), _rows([9]), _rows([3, 3]), _rows([5], nan), _rows([5], INF), _rows([5], -1.0),
                _rows([5], 0.2, nan), _rows([5], 0.2, -1.0)):
        r = np.ascontiguousarray(bad)
        assert g.lib.nb_upload_ccd_bodies(g.ctx, r.ctypes.data_as(ctypes.c_void_p), len(r), g.stream) == NB_ERR_ARGUMENT
        assert g.download_ccd_bodies().tobytes() == good.tobytes()
    assert g.lib.nb_upload_ccd_bodies(g.ctx, None, 1, g.stream) == NB_ERR_ARGUMENT
    assert _state(g) == before and g.download_ccd_bodies().tobytes() == good.tobytes()
    # nb_advance with a set and no collide since the last advance launches nothing
    g.step_staged()
    before, launches = _state(g), g.launch_count()
    with pytest.raises(nudge_b200.NudgeError, match="nb_collide since the last nb_advance"):
        g.advance()
    assert _state(g) == before and g.launch_count() == launches
    # a sharded context refuses the upload, and nb_shard_step a context with a set
    b = nudge_b200.Sim(s)
    b.upload_ccd_bodies(good)
    b.shard_create(0, 1, None, 1, 1)
    with pytest.raises(nudge_b200.NudgeError, match="continuous collision"):
        b.shard_step("peer")
    with pytest.raises(nudge_b200.NudgeError, match="nb_shard_create"):
        b.upload_ccd_bodies(_rows([5]))


def test_in_scene_casts_record_no_fallbacks(mixed):
    for scene, settle in (mixed, (small_mixed_scene(), 150)):
        g = _settled(scene, settle)
        bodies = np.arange(1, scene.n_bodies, dtype=np.uint32)
        g.upload_ccd_bodies(_rows(bodies, 0.1))
        _fire(g, bodies[::7], np.random.default_rng(2), 50.0)
        for _ in range(20):
            g.step()
        assert g.debug_scalar("ccd_fallbacks") == 0
        if scene is not mixed[0]:
            assert g.debug_scalar("grid_level") <= 8
