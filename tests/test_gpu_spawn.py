"""Spawning and despawning on the device (nb_add_bodies, nb_remove_bodies; DESIGN.md section 8.10) against the host edit they replace: a twin
context edited through download -> tests/spawn_ref.py -> re-upload of bodies, colliders, connections, filters, sensors, kinematic set and user
rows saves byte-identical state files right after every edit and stays byte-identical over a run that sleeps and wakes (nb_step graph replay
and stage calls); contact events equal the twin's and sensor events the restatement's; the 1,500-box drop after an edit equals the oracle on
the restated scene at every stage; a removal wakes the stack above and leaves another pile asleep; tag reuse; argument errors; launch counts
and graph replay; the Python mirrors."""
import ctypes
import os
import tempfile
import numpy as np
import pytest
import nudge_b200
from nudge_b200 import scenes, abi, ROW
from tests.spawn_ref import REMOVED, add_bodies, rebuild_oracle, remove_bodies, live_scene
from tests.parity_util import Report, compare_oracle_gpu_step
from tests.gpu_util import side_stream
from tests.test_body_impulse_oracle import two_piles, settle_and_sleep

pytestmark = pytest.mark.gpu
NB_ERR_CAPACITY, NB_ERR_ARGUMENT = -2, -3
SENSOR_PAIRS = 4096
SPARE = 400


def _state(x):
    x.download_bodies(); x.download_contacts(); x.download_cache()
    c = x.contacts_view()
    parts = [x.transforms, x.momentum, x.idle, c["data"], c["bodies"], c["tags"], c["features"], c["sleeping"], c["active"]]
    cv = x.cache_view()
    return b"".join(np.ascontiguousarray(a).tobytes() for a in parts + [cv["tags"], cv["features"], cv["data"]])


def _counts(x):
    c = x.counts()
    return (c.pairs, c.live_pairs, c.contacts, c.sleeping, c.active, c.cache, c.culled, c.batches, c.levels, c.overflow)


def _saved(x):
    with tempfile.TemporaryDirectory() as d:
        p = os.path.join(d, "s.nbstate")
        x.save_state(p)
        return open(p, "rb").read()


def _ball_rows(pairs):
    """Three point-to-point rows (x, y, z) per joined pair."""
    rows = np.zeros(3 * len(pairs), ROW)
    for j, (a, b) in enumerate(pairs):
        for k in range(3):
            r = rows[3 * j + k]
            r["a"], r["b"] = a, b
            r["lin_a"][k], r["lin_b"][k] = 1.0, -1.0
            r["lo"], r["hi"] = -np.inf, np.inf
    return rows


def _scene(seed=31):
    """Boxes and spheres falling on the ground, three sensor zones on body 0, a filter table, a kinematic slab, ball joints and connections."""
    rng = np.random.default_rng(seed)
    s = scenes.demo_scene(150, 150, iterations=4, spread=6.0, height=8.0, seed=seed)
    zones = np.array([(-3.0, 4.0, 0.0), (3.0, 4.0, 2.0), (0.0, 4.0, -3.0)], np.float32)
    nb = s.n_boxes
    tags0 = int(max(s.box_tags.max(), s.sphere_tags.max())) + 1
    z = np.zeros(3, scenes.TRANSFORM); z["rotation"][:, 3] = 1; z["position"] = zones
    zb = np.zeros(3, scenes.BOX); zb["size"] = (2.0, 4.0, 2.0)
    s.box_tags = np.concatenate([s.box_tags, tags0 + np.arange(3, dtype=np.uint32)])
    s.box_data = np.concatenate([s.box_data, zb]); s.box_transforms = np.concatenate([s.box_transforms, z])
    K = s.n_colliders
    s.sensors = np.zeros(K, np.uint8); s.sensors[nb:nb + 3] = 1
    s.collision_filters = np.zeros(K, scenes.FILTER)
    s.collision_filters["category"] = 1 << rng.integers(0, 3, K)
    s.collision_filters["mask"] = 0xffff
    s.collision_filters["mask"][rng.random(K) < 0.1] = 0xfffe   # a few colliders ignore category 1
    s.filter_flags = scenes.FILTER_SKIP_CONNECTED
    s.kinematic = np.array([(7, (0.0, 0.0, 0.0), (0.0, 0.0, 0.0), 0)], scenes.KINEMATIC)
    s.transforms["position"][7] = (0.0, -9.0, 0.0)
    pairs = [(10, 11), (20, 21), (30, 0), (40, 41), (41, 42)]
    s.connections = np.array(pairs + [(60, 61), (70, 80)], scenes.PAIR32)
    return s, _ball_rows(pairs)


def _sim(s, rows, stream=0):
    x = nudge_b200.Sim(s, stream=stream, max_bodies=s.n_bodies + SPARE, max_boxes=s.n_boxes + SPARE, max_spheres=s.n_spheres + SPARE)
    x.upload_sensors(s.sensors, SENSOR_PAIRS)
    x.upload_constraint_rows(rows)
    return x


def _reupload(x, new, rows):
    """The host round trip's upload of everything the edit changes."""
    x.scene = new
    abi.HostState.__init__(x, new, x.cap)
    L, ctx, st = x.lib, x.ctx, x.stream
    x._ck(L.nb_upload_bodies(ctx, ctypes.byref(x.bodies), st), "nb_upload_bodies")
    x._ck(L.nb_upload_colliders(ctx, ctypes.byref(x.colliders), st), "nb_upload_colliders")
    x._ck(L.nb_upload_connections(ctx, ctypes.byref(x.conn), st), "nb_upload_connections")
    x.upload_collision_filters(new.collision_filters, new.filter_flags)
    x.upload_sensors(new.sensors, SENSOR_PAIRS)
    k = None
    if new.kinematic is not None:
        k = new.kinematic.copy()
        b = k["body"].astype(np.int64)
        k["velocity"] = new.momentum["velocity"][b]; k["angular_velocity"] = new.momentum["angular_velocity"][b]
    x.upload_kinematic_bodies(k)
    x.upload_constraint_rows(rows)


def _twin_remove(t, idx, nrows):
    t.download_bodies(); t.download_cache()
    rows = t.download_constraint_rows(nrows)
    new, new_rows, _, woken = remove_bodies(live_scene(t), idx, t.cache_view()["tags"], rows)
    _reupload(t, new, new_rows)
    return len(new_rows), woken


def _twin_add(t, fr, nrows):
    t.download_bodies()
    rows = t.download_constraint_rows(nrows)
    _reupload(t, add_bodies(live_scene(t), fr), rows)


def _fragment(rng, n, first_tag):
    """n bodies (boxes, then spheres) dropped beside the pile, with their filter and sensor table entries."""
    nb = n // 2
    fb = scenes.fragment(rng.uniform(-5, 5, (nb, 3)) + (25, 0, 0), "box", rng.uniform(0.3, 0.7, (nb, 3)), first_tag)
    fs = scenes.fragment(rng.uniform(-5, 5, (n - nb, 3)) + (25, 0, 0), "sphere", rng.uniform(0.3, 0.7, n - nb), first_tag + nb)
    fr = scenes.Scene(0, 0, 0)
    for k in ("transforms", "properties", "momentum", "idle"):
        setattr(fr, k, np.concatenate([getattr(fb, k), getattr(fs, k)]))
    fr.box_tags, fr.box_data, fr.box_transforms = fb.box_tags, fb.box_data, fb.box_transforms
    sx = fs.sphere_transforms.copy(); sx["body"] += np.uint32(nb)
    fr.sphere_tags, fr.sphere_data, fr.sphere_transforms = fs.sphere_tags, fs.sphere_data, sx
    K = fr.n_colliders
    fr.collision_filters = np.zeros(K, scenes.FILTER); fr.collision_filters["category"] = 1 << rng.integers(0, 3, K); fr.collision_filters["mask"] = 0xffff
    fr.sensors = np.zeros(K, np.uint8)
    return fr


def _pick(rng, B, kin, n):
    pool = np.setdiff1d(np.arange(1, B), kin)
    return rng.choice(pool, n, replace=False).astype(np.uint32)


def _kin(x):
    return [] if x.scene.kinematic is None else x.scene.kinematic["body"].tolist()


@pytest.mark.parametrize("mode", ["graph", "staged"])
def test_device_edit_equals_the_host_round_trip_bit_for_bit(mode):
    s, rows = _scene()
    dev, twin = _sim(s, rows, side_stream()), _sim(s, rows, side_stream())
    for x in (dev, twin):
        x.enable_contact_events(1 << 16)
    rng = np.random.default_rng(3)
    nrows = len(rows)
    tag = 100000
    edits = sleeping = 0
    for i in range(76):
        if i == 30:   # the whole scene asleep, identically in both: the edits then wake parts of it
            for x in (dev, twin):
                x.download_bodies(); x.idle[1:] = 0xff
                x.momentum["velocity"][1:] = 0; x.momentum["angular_velocity"][1:] = 0
                x.upload_bodies()
        if i % 9 == 4:
            idx = _pick(rng, dev.scene.n_bodies, _kin(dev), int(rng.integers(1, 12)))
            if i == 58:   # a joined body: its rows and connection go
                idx = np.unique(np.concatenate([idx, dev.download_constraint_rows(nrows)["a"][:1]])).astype(np.uint32)
            if i == 67:   # the kinematic slab: the set becomes empty
                idx = np.unique(np.concatenate([idx, _kin(dev)])).astype(np.uint32)
            dev.remove_bodies(idx)
            nrows, _ = _twin_remove(twin, idx, nrows)
            edits += 1
            assert _saved(dev) == _saved(twin), i
        if i % 11 == 7:
            fr = _fragment(rng, int(rng.integers(1, 10)), tag)
            tag += 20
            dev.add_bodies(fr, filters=fr.collision_filters, sensors=fr.sensors)
            _twin_add(twin, fr, nrows)
            edits += 1
            assert _saved(dev) == _saved(twin), i
        if mode == "graph":
            dev.step(); twin.step()
        else:
            dev.step_staged(); twin.step_staged()
        assert _state(dev) == _state(twin), (mode, i)
        cd = _counts(dev)
        assert cd == _counts(twin), (mode, i)
        sleeping += cd[3]
        ed, et = dev.contact_events()[0], twin.contact_events()[0]
        contact = lambda e: e[e["kind"] <= scenes.CONTACT_END].tobytes()
        assert contact(ed) == contact(et), (mode, i)
        assert np.array_equal(dev.download_constraint_rows(nrows), twin.download_constraint_rows(nrows)), i
    assert edits >= 14 and sleeping > 0 and nrows < len(rows) and dev.scene.kinematic is None


def test_throughput_mode_edit_equals_the_host_round_trip():
    """Throughput mode: its impulses vary from run to run, so before every edit the twin takes the device context's state (state file and
    user rows); the edited states must then be byte-identical and the next step must agree up to that run-to-run noise.  The solver's
    per-body accumulator holds the gathered momentum rows during a removal and must be left all zeros."""
    s, rows = _scene(37)
    dev, twin = _sim(s, rows, side_stream()), _sim(s, rows, side_stream())
    for x in (dev, twin):
        x.set_solver_mode("throughput")
    rng = np.random.default_rng(4)
    nrows = len(rows)
    tag = 400000
    checked = 0
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "dev.nbstate")
        for i in range(72):
            if i == 30:
                dev.download_bodies(); dev.idle[1:] = 0xff
                dev.momentum["velocity"][1:] = 0; dev.momentum["angular_velocity"][1:] = 0
                dev.upload_bodies()
            remove, add = i % 9 == 4, i % 11 == 7
            if remove or add:
                dev.save_state(path); twin.load_state(path)
                abi.HostState.__init__(twin, dev.scene.copy(), twin.cap)
                twin.upload_constraint_rows(dev.download_constraint_rows(nrows))
            if remove:
                idx = _pick(rng, dev.scene.n_bodies, _kin(dev), int(rng.integers(1, 12)))
                dev.remove_bodies(idx)
                nrows, _ = _twin_remove(twin, idx, nrows)
            if add:
                fr = _fragment(rng, int(rng.integers(1, 10)), tag)
                tag += 20
                dev.add_bodies(fr, filters=fr.collision_filters, sensors=fr.sensors)
                _twin_add(twin, fr, nrows)
            if remove or add:
                assert _saved(dev) == _saved(twin), i
            dev.step()
            if remove or add:
                twin.step()
                dev.download_bodies(); twin.download_bodies()
                for f in ("velocity", "angular_velocity"):
                    assert np.allclose(dev.momentum[f], twin.momentum[f], rtol=1e-3, atol=1e-3), (i, f)
                assert np.allclose(dev.transforms["position"], twin.transforms["position"], rtol=1e-4, atol=1e-4), i
                assert np.abs(dev.momentum["velocity"]).max() > 0.1 or i > 30, i   # something moves, so a corruption would show
                checked += 1
    assert checked == 13   # the steps with an edit: 8 removals and 6 additions, one step with both


def test_sensor_events_follow_the_remapped_overlap_list():
    s, rows = _scene(32)
    g = _sim(s, rows, side_stream())
    g.enable_contact_events(1 << 16)
    for _ in range(60):
        g.step()
    g.contact_events()
    ov = g.sensor_overlaps()
    assert len(ov) > 4
    bodies = np.unique(np.concatenate([ov["body_a"], ov["body_b"]]))
    victims = np.setdiff1d(bodies, [0] + _kin(g))[:3].astype(np.uint32)
    _, _, want_old, _ = remove_bodies(s, victims, None, None, ov)
    g.remove_bodies(victims)
    g.step()
    ev = g.contact_events()[0]
    cur = g.sensor_overlaps()
    sens = ev[ev["kind"] >= scenes.SENSOR_BEGIN]
    old_k, cur_k = set(want_old["tags"].tolist()), set(cur["tags"].tolist())
    assert len(old_k & cur_k) > 0   # kept overlaps: no BEGIN for them (checked by the equality below)
    want = sorted([(t, scenes.SENSOR_END, a, b) for t, a, b in want_old[["tags", "body_a", "body_b"]].tolist() if t not in cur_k] +
                  [(t, scenes.SENSOR_BEGIN, a, b) for t, a, b in cur[["tags", "body_a", "body_b"]].tolist() if t not in old_k])
    got = sorted(sens[["tags", "kind", "body_a", "body_b"]].tolist())
    assert got == want
    ends = [e for e in got if e[1] == scenes.SENSOR_END]
    assert any(REMOVED in (e[2], e[3]) for e in ends)   # the removed bodies' overlaps end, with NB_REMOVED_BODY


def test_oracle_on_the_restated_scene_equals_the_device_at_every_stage():
    from oracle import pyoracle
    s = scenes.box_drop(1500, iterations=8)
    o = pyoracle.OracleSim(s)
    g = nudge_b200.Sim(s, contact_capacity=o.cap, debug=True, max_bodies=s.n_bodies + 50, max_boxes=s.n_boxes + 50)
    rng = np.random.default_rng(6)
    for i in range(14):
        if i == 4:
            idx = rng.choice(np.arange(1, s.n_bodies), 40, replace=False).astype(np.uint32)
            fr = scenes.fragment(rng.uniform(-8, 8, (40, 3)) + (0, 14, 0), "box", rng.uniform(0.4, 0.8, (40, 3)), 50000)
            g.remove_bodies(idx); g.add_bodies(fr)
            new = add_bodies(remove_bodies(live_scene(o), idx, o.cache_tags[:o.cache.count])[0], fr)
            o = rebuild_oracle(o, new)
            g.download_bodies()
            assert g.transforms.tobytes() == o.transforms.tobytes() and g.idle.tobytes() == o.idle.tobytes()
        rep = Report("step %d" % i)
        assert compare_oracle_gpu_step(o, g, rep), str(rep)


def test_removing_a_lower_crate_wakes_the_stack_above_and_not_the_other_pile():
    s, pile_a, pile_b = two_piles()
    g = nudge_b200.Sim(s, stream=side_stream())
    settle_and_sleep(g)
    g.step()
    g.collide(); g.download_contacts()
    assert g.counts().active == 0
    g.apply_gravity_damping(); g.read_cached_impulses(); g.setup_contact_constraints(); g.apply_impulses(8)
    g.update_cached_impulses(); g.write_cached_impulses(); g.advance()
    g.download_bodies()
    moved = lambda b: int(b) - (1 if b > pile_a[1] else 0)
    before_b = g.transforms[pile_b].tobytes()
    top_y = g.transforms["position"][pile_a[-2], 1]
    g.remove_bodies([pile_a[1]])
    g.download_bodies()
    assert g.idle[moved(pile_a[2])] == 0 and g.idle[moved(pile_a[0])] == 0 and (g.idle[[moved(b) for b in pile_b]] == 0xff).all()
    g.collide(); g.download_contacts()
    assert sorted(g.contacts_view()["active"].tolist()) == sorted(moved(b) for b in pile_a if b != pile_a[1])
    g.apply_gravity_damping(); g.read_cached_impulses(); g.setup_contact_constraints(); g.apply_impulses(8)
    g.update_cached_impulses(); g.write_cached_impulses(); g.advance()
    for _ in range(90):
        g.step()
    g.download_bodies()
    assert g.transforms[[moved(b) for b in pile_b]].tobytes() == before_b
    assert g.transforms["position"][moved(pile_a[-2]), 1] < top_y - 0.5   # the stack above fell into the gap


def test_a_removed_tag_reused_before_the_next_step_behaves_like_the_twin():
    s, rows = _scene(33)
    dev, twin = _sim(s, rows, side_stream()), _sim(s, rows, side_stream())
    for _ in range(40):
        dev.step(); twin.step()
    victim = 120
    bi = list(dev.scene.box_transforms["body"]).index(victim)
    tag = int(dev.scene.box_tags[bi])
    dev.remove_bodies([victim])
    nrows, _ = _twin_remove(twin, [victim], len(rows))
    fr = scenes.fragment(s.transforms["position"][victim:victim + 1], "box", s.box_data["size"][bi:bi + 1], tag)
    fr.collision_filters = np.array([(1, 0xffff)], scenes.FILTER); fr.sensors = np.zeros(1, np.uint8)
    dev.add_bodies(fr, filters=fr.collision_filters, sensors=fr.sensors)
    _twin_add(twin, fr, nrows)
    assert _saved(dev) == _saved(twin)
    for i in range(10):
        dev.step(); twin.step()
        assert _state(dev) == _state(twin), i


def test_argument_errors_and_no_ops_change_nothing():
    s, rows = _scene(34)
    g = _sim(s, rows)
    g.step_staged()
    before = _saved(g)
    B = g.scene.n_bodies
    L, ctx, st = g.lib, g.ctx, g.stream
    arr = lambda *v: np.ascontiguousarray(np.array(v, np.uint32))
    for bad in (arr(0, 3), arr(5, B), arr(4, 9, 4)):
        assert L.nb_remove_bodies(ctx, abi.ptr(bad), len(bad), st) == NB_ERR_ARGUMENT
    assert L.nb_remove_bodies(ctx, None, 2, st) == NB_ERR_ARGUMENT
    c0 = g.launch_count()
    assert L.nb_remove_bodies(ctx, None, 0, st) == 0 and g.launch_count() == c0
    fr = scenes.fragment([(0, 20, 0)], "box", first_tag=90000)
    P = lambda a: abi.ptr(np.ascontiguousarray(a))
    parts = [np.ascontiguousarray(a) for a in (fr.transforms, fr.properties, fr.momentum, fr.idle, fr.box_tags, fr.box_data, fr.box_transforms)]
    bodies = abi.BodyData(*(abi.ptr(p) for p in parts[:4]), 1)
    cols = abi.ColliderData(abi.Shapes(abi.ptr(parts[4]), abi.ptr(parts[5]), abi.ptr(parts[6]), 1), abi.Shapes(None, None, None, 0))
    f1, s1 = np.zeros(1, scenes.FILTER), np.zeros(1, np.uint8)
    both = nudge_b200.SpawnTables(P(f1), P(s1))
    assert L.nb_add_bodies(ctx, ctypes.byref(bodies), ctypes.byref(cols), None, st) == NB_ERR_ARGUMENT                      # tables missing
    assert L.nb_add_bodies(ctx, ctypes.byref(bodies), ctypes.byref(cols), ctypes.byref(nudge_b200.SpawnTables(P(f1), None)), st) == NB_ERR_ARGUMENT
    big = abi.BodyData(*(abi.ptr(p) for p in parts[:4]), SPARE + 1)
    assert L.nb_add_bodies(ctx, ctypes.byref(big), None, None, st) == NB_ERR_CAPACITY
    many = abi.Shapes(abi.ptr(parts[4]), abi.ptr(parts[5]), abi.ptr(parts[6]), SPARE + 1)
    none = abi.Shapes(None, None, None, 0)
    for cols_big in (abi.ColliderData(many, none), abi.ColliderData(none, many)):   # max_boxes, then max_spheres
        assert L.nb_add_bodies(ctx, None, ctypes.byref(cols_big), ctypes.byref(both), st) == NB_ERR_CAPACITY
    parts[6]["body"] = B + 1
    assert L.nb_add_bodies(ctx, ctypes.byref(bodies), ctypes.byref(cols), ctypes.byref(both), st) == NB_ERR_ARGUMENT     # body beyond B + 1
    assert _saved(g) == before
    # superfluous tables on a context without them
    p = nudge_b200.Sim(scenes.demo_scene(20, 20, seed=3), max_bodies=100, max_boxes=100)
    parts[6]["body"] = 0
    assert p.lib.nb_add_bodies(p.ctx, ctypes.byref(bodies), ctypes.byref(cols), ctypes.byref(both), p.stream) == NB_ERR_ARGUMENT
    assert p.lib.nb_add_bodies(p.ctx, ctypes.byref(bodies), ctypes.byref(cols), None, p.stream) == 0
    # stage calls between an edit and the next collide are refused; the collide lifts it
    g.remove_bodies([5])
    for call in (g.read_cached_impulses, g.setup_contact_constraints, g.apply_impulses, g.update_cached_impulses, g.write_cached_impulses, g.advance):
        with pytest.raises(nudge_b200.NudgeError, match="edited"):
            call()
    # a state file replaces the edited scene: the stage calls are legal again
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "g.nbstate")
        g.save_state(path)
        saved_scene = g.scene.copy()
        g.remove_bodies([6])
        with pytest.raises(nudge_b200.NudgeError, match="edited"):
            g.read_cached_impulses()
        g.load_state(path)
        abi.HostState.__init__(g, saved_scene, g.cap)
        g.read_cached_impulses()
    g.step_staged()
    # a row or a connection naming a body at or beyond the body count (their uploads accept it) is refused, changing nothing
    Bp = p.scene.n_bodies
    row = np.zeros(1, ROW); row["a"] = Bp + 3
    p.upload_constraint_rows(row)
    before_p = _saved(p)
    assert p.lib.nb_remove_bodies(p.ctx, abi.ptr(arr(2)), 1, p.stream) == NB_ERR_ARGUMENT
    assert _saved(p) == before_p
    p.upload_constraint_rows(np.zeros(0, ROW))
    far = np.array([(Bp + 2, 1)], scenes.PAIR32)
    p._ck(p.lib.nb_upload_connections(p.ctx, ctypes.byref(abi.Connections(abi.ptr(far), 1)), p.stream), "nb_upload_connections")
    before_p = _saved(p)
    assert p.lib.nb_remove_bodies(p.ctx, abi.ptr(arr(2)), 1, p.stream) == NB_ERR_ARGUMENT
    assert _saved(p) == before_p
    # a shard context refuses both
    g.shard_create(0, 1, None, 16, 16)
    assert L.nb_remove_bodies(ctx, abi.ptr(arr(3)), 1, st) == NB_ERR_ARGUMENT
    assert L.nb_add_bodies(ctx, ctypes.byref(bodies), None, None, st) == NB_ERR_ARGUMENT


def test_launches_per_step_equal_a_fresh_context_and_graph_replay_equals_plain_launches():
    s, _ = _scene(35)
    none = np.zeros(0, ROW)
    a, p = _sim(s, none, side_stream()), _sim(s, none)   # p: the legacy default stream, plain launches
    rng = np.random.default_rng(12)
    tag = 200000
    for i in range(12):
        idx = _pick(rng, a.scene.n_bodies, _kin(a), 5)
        c0 = a.launch_count()
        a.remove_bodies(idx); p.remove_bodies(idx)
        assert 8 <= a.launch_count() - c0 <= 14, i
        fr = _fragment(rng, 4, tag); tag += 10
        c0 = a.launch_count()
        a.add_bodies(fr, filters=fr.collision_filters, sensors=fr.sensors); p.add_bodies(fr, filters=fr.collision_filters, sensors=fr.sensors)
        assert a.launch_count() == c0, i
        a.step(); p.step()
        assert _state(a) == _state(p), i
    assert a.debug_scalar("graph_active") == 1
    a.download_bodies()
    fresh = _sim(live_scene(a), none, side_stream())
    per_step = []
    for x in (a, fresh):
        c0 = x.launch_count(); x.step(); c1 = x.launch_count(); x.step()
        per_step.append((c1 - c0, x.launch_count() - c1))
    assert per_step[0] == per_step[1]


def test_python_mirrors_describe_the_device():
    s, rows = _scene(36)
    g = _sim(s, rows, side_stream())
    for _ in range(10):
        g.step()
    g.download_bodies(); g.download_cache()
    want, _, _, _ = remove_bodies(live_scene(g), [3, 50, 200], g.cache_view()["tags"])
    g.remove_bodies([3, 50, 200])
    fr = _fragment(np.random.default_rng(2), 6, 300000)
    want = add_bodies(want, fr)
    g.add_bodies(fr, filters=fr.collision_filters, sensors=fr.sensors)
    got = g.scene
    for k in ("properties", "box_tags", "box_data", "box_transforms", "sphere_tags", "sphere_data", "sphere_transforms", "connections", "collision_filters", "sensors"):
        assert getattr(got, k).tobytes() == getattr(want, k).tobytes(), k
    assert got.kinematic["body"].tolist() == want.kinematic["body"].tolist()
    cols = g.download_colliders()
    for k, v in cols.items():
        assert v.tobytes() == getattr(want, k).tobytes(), k
    assert g.download_connections().tobytes() == want.connections.tobytes()
    g.download_bodies()
    assert g.idle.tobytes() == want.idle.tobytes() and g.transforms.tobytes() == want.transforms.tobytes()
    g.step()
    g.upload()   # the mirrors re-upload cleanly
    g.step()
