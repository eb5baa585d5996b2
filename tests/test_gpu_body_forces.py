"""Per-body forces on the device (nb_set_body_forces, nb_clear_body_forces, nb_download_body_forces; DESIGN.md section 8.11): a table of
default entries is no table; the oracle with the restated stage (tests/body_force_ref.py) at every stage; the stage call in throughput
mode; waking and keeping awake; graph replay with entries changed every step; spawn and despawn against the host round trip; state files
and nb_replay; nb_upload_bodies, kinematic bodies and nb_shard_step; and the argument errors."""
import ctypes, os, struct, subprocess, tempfile
import numpy as np
import pytest
import nudge_b200
from nudge_b200 import scenes
from tests.body_force_ref import BodyForceOracleSim, apply_stage, default_table, remove_table, add_table, set_entries
from tests.parity_util import Report, compare_oracle_gpu_step
from tests.gpu_util import side_stream, fnv1a
from tests.test_body_impulse_oracle import two_piles, settle_and_sleep
from tests.test_gpu_spawn import _scene, _sim, _twin_remove, _twin_add, _fragment, _pick, _kin, _saved, _state, _counts

pytestmark = pytest.mark.gpu
NB_ERR_CAPACITY, NB_ERR_ARGUMENT = -2, -3
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F = np.float32


def _random_entries(rng, bodies, local=0.5):
    """BODY_FORCE rows for `bodies`: gravity scale in [-0.5, 2], damping, world or body-frame forces and torques, some of them zero."""
    b = np.asarray(bodies, np.uint32)
    r = scenes.default_body_forces(b)
    n = len(b)
    r["gravity_scale"] = rng.uniform(-0.5, 2.0, n)
    r["linear_damping"] = rng.uniform(0.0, 2.0, n) * (rng.random(n) < 0.6)
    r["angular_damping"] = rng.uniform(0.0, 2.0, n) * (rng.random(n) < 0.6)
    r["force"] = rng.normal(0.0, 8.0, (n, 3)) * (rng.random((n, 1)) < 0.5)
    r["torque"] = rng.normal(0.0, 2.0, (n, 3)) * (rng.random((n, 1)) < 0.4)
    r["flags"] = (rng.random(n) < local) * scenes.BODY_FORCE_LOCAL
    return r


def _mixed(n, seed):
    s = scenes.demo_scene(n // 2, n - n // 2, iterations=4, spread=12.0, height=20.0, seed=seed)
    s.transforms["rotation"][1:] = scenes._random_unit_quaternions(np.random.default_rng(seed), s.n_bodies - 1)
    return s


def _set(lib_sim, rows):
    r = np.ascontiguousarray(rows, scenes.BODY_FORCE)
    return lib_sim.lib.nb_set_body_forces(lib_sim.ctx, r.ctypes.data_as(ctypes.c_void_p) if len(r) else None, len(r), lib_sim.stream)


def _header(raw):
    return struct.unpack_from("<I", raw, 8)[0], struct.unpack_from("<8I", raw, 36)


def test_a_table_of_default_entries_is_no_table():
    s, pile_a, pile_b = two_piles()
    for graph in (True, False):
        a = nudge_b200.Sim(s, stream=side_stream() if graph else 0)
        b = nudge_b200.Sim(s, stream=side_stream() if graph else 0)
        b.set_body_forces(scenes.default_body_forces(np.arange(1, s.n_bodies, 2)))
        settle_and_sleep(a, 40); settle_and_sleep(b, 40)   # both asleep with the same rows (the set woke its bodies)
        per_step, sleeping = [], 0
        for i in range(60):
            if i == 25:   # wake pile a in both
                hit = np.zeros(1, scenes.BODY_IMPULSE); hit["body"] = pile_a[1]; hit["impulse"] = (0.3, 0.0, 0.0)
                a.apply_body_impulses(hit); b.apply_body_impulses(hit)
            la, lb = a.launch_count(), b.launch_count()
            if graph:
                a.step(); b.step()
            else:
                a.step_staged(); b.step_staged()
            per_step.append((a.launch_count() - la, b.launch_count() - lb))
            assert _state(a) == _state(b), (graph, i)
            assert _counts(a) == _counts(b), (graph, i)
            sleeping += _counts(a)[3]
        assert all(x == y for x, y in per_step), per_step
        assert sleeping > 0
        ra, rb = _saved(a), _saved(b)
        va, resa = _header(ra); vb, resb = _header(rb)
        assert va == 1 and vb == 5 and resb[5] == 1
        table = default_table(s.n_bodies).tobytes()
        assert rb[len(ra):] == table and rb[12:36] == ra[12:36] and rb[68:len(ra)] == ra[68:]
        assert np.array_equal(b.download_body_forces(), default_table(s.n_bodies)) and np.array_equal(a.download_body_forces(), default_table(s.n_bodies))


def test_stage_parity_with_random_entries_against_the_restated_oracle():
    s = _mixed(1500, 41)
    o = BodyForceOracleSim(s)
    g = nudge_b200.Sim(s, contact_capacity=o.cap, debug=True)
    rng = np.random.default_rng(5)
    rows = _random_entries(rng, np.arange(1, s.n_bodies))
    o.set_body_forces(rows); g.set_body_forces(rows)
    for i in range(16):
        if i % 4 == 3:   # re-draw some entries between steps
            redo = _random_entries(rng, rng.choice(np.arange(1, s.n_bodies), 200, replace=False))
            o.set_body_forces(redo); g.set_body_forces(redo)
        rep = Report("body forces step %d" % i)
        assert compare_oracle_gpu_step(o, g, rep), str(rep)
    assert np.array_equal(g.download_body_forces(), o.table)


def test_throughput_stage_call_equals_the_restatement():
    s = _mixed(1500, 42)
    g = nudge_b200.Sim(s)
    g.set_solver_mode("throughput")
    rng = np.random.default_rng(6)
    table = default_table(s.n_bodies)
    for i in range(12):
        rows = _random_entries(rng, rng.choice(np.arange(1, s.n_bodies), 500, replace=False))
        g.set_body_forces(rows); set_entries(table, rows)
        g.collide()
        g.download_contacts(); g.download_bodies()
        active = g.contacts_view()["active"]
        want = _host_copy(g)
        apply_stage(want, table, active, s.time_step, s.gravity, s.damping)
        g.apply_gravity_damping()
        g.download_bodies()
        assert g.momentum.tobytes() == want.momentum.tobytes() and g.idle.tobytes() == want.idle.tobytes(), i
        g.read_cached_impulses(); g.setup_contact_constraints(); g.apply_impulses(int(s.iterations))
        g.update_cached_impulses(); g.write_cached_impulses(); g.advance()


def _host_copy(x):
    import types
    return types.SimpleNamespace(transforms=x.transforms.copy(), properties=x.properties.copy(), momentum=x.momentum.copy(), idle=x.idle.copy())


def _active(g):
    g.collide(); g.download_contacts()
    return set(g.contacts_view()["active"].tolist())


def _finish(g):
    g.apply_gravity_damping(); g.read_cached_impulses(); g.setup_contact_constraints(); g.apply_impulses(int(g.scene.iterations))
    g.update_cached_impulses(); g.write_cached_impulses(); g.advance()


def test_gravity_scale_wakes_the_island_and_a_force_keeps_it_awake():
    s, pile_a, pile_b = two_piles()
    g = nudge_b200.Sim(s)
    settle_and_sleep(g)
    assert _active(g) == set()
    _finish(g)
    up = scenes.default_body_forces([pile_a[-1]]); up["gravity_scale"] = -1.0   # the sphere on top of pile a
    g.set_body_forces(up)
    g.download_bodies()
    assert g.idle[pile_a[-1]] == 0 and (g.idle[pile_b] == 0xff).all()
    assert _active(g) == set(pile_a.tolist())
    y0 = float(g.transforms["position"][pile_a[-1], 1])
    _finish(g)
    for _ in range(30):
        g.step_staged()
    g.download_bodies()
    assert float(g.transforms["position"][pile_a[-1], 1]) > y0 + 0.1
    # a downward force on the bottom box of pile b: awake for as long as it carries it, asleep again after it is cleared
    press = scenes.default_body_forces([pile_b[0]]); press["force"] = (0.0, -30.0, 0.0)
    g.set_body_forces(press)
    for i in range(300):
        assert pile_b[0] in _active(g), i
        _finish(g)
    g.set_body_forces(scenes.default_body_forces([pile_b[0]]))
    for i in range(800):
        if pile_b[0] not in _active(g):
            break
        _finish(g)
    else:
        raise AssertionError("pile b never fell asleep after its force was cleared")


def test_graph_replay_with_entries_changed_every_step_equals_plain_launches():
    s = _mixed(600, 43)
    a, b = nudge_b200.Sim(s, stream=side_stream()), nudge_b200.Sim(s)   # graph replay / plain launches on the legacy stream
    rng = np.random.default_rng(7)
    a.step(); b.step()
    before = a.launch_count(); a.step(); b.step(); no_table = a.launch_count() - before
    rows = _random_entries(rng, np.arange(1, s.n_bodies))
    a.set_body_forces(rows); b.set_body_forces(rows)   # creates the table: the graph re-records with k_body_forces
    for i in range(30):
        r = _random_entries(rng, rng.choice(np.arange(1, s.n_bodies), 50, replace=False))
        a.set_body_forces(r); b.set_body_forces(r)
        before = a.launch_count()
        a.step(); b.step()
        if i:
            assert a.launch_count() - before == no_table, i   # the replayed step; the scatter ran before
        assert _state(a) == _state(b), i
    assert a.debug_scalar("graph_active") == 1
    a.clear_body_forces(); b.clear_body_forces()   # re-records without it
    for i in range(5):
        before = a.launch_count()
        a.step(); b.step()
        assert a.launch_count() - before == no_table
        assert _state(a) == _state(b), i


def _twin_forces(t, table):
    """The host round trip's body force upload: every non-default entry, then the body rows again (nb_set_body_forces wakes its bodies)."""
    d = default_table(len(table))
    nd = table[[table[i].tobytes() != d[i].tobytes() for i in range(len(table))]]
    t.clear_body_forces()
    t.set_body_forces(nd)
    t.upload_bodies()


def test_spawn_and_despawn_move_the_entries_like_the_host_round_trip():
    s, rows = _scene()
    dev, twin = _sim(s, rows, side_stream()), _sim(s, rows, side_stream())
    rng = np.random.default_rng(8)
    ent = _random_entries(rng, np.setdiff1d(np.arange(1, s.n_bodies), _kin(dev))[::3])
    table = default_table(s.n_bodies); set_entries(table, ent)
    for x in (dev, twin):
        x.set_body_forces(ent)
    nrows, tag, edits = len(rows), 100000, 0
    for i in range(40):
        if i % 9 == 4:
            idx = _pick(rng, dev.scene.n_bodies, _kin(dev), int(rng.integers(1, 12)))
            dev.remove_bodies(idx)
            nrows, _ = _twin_remove(twin, idx, nrows)
            table = remove_table(table, idx)
            _twin_forces(twin, table)
            edits += 1
        if i % 11 == 7:
            fr = _fragment(rng, int(rng.integers(1, 10)), tag)
            tag += 20
            B0 = dev.scene.n_bodies
            dev.add_bodies(fr, filters=fr.collision_filters, sensors=fr.sensors)
            _twin_add(twin, fr, nrows)
            table = add_table(table, fr.n_bodies)
            _twin_forces(twin, table)
            assert np.array_equal(dev.download_body_forces()[B0:], default_table(dev.scene.n_bodies)[B0:])
            edits += 1
        if i % 11 == 7 or i % 9 == 4:
            assert np.array_equal(dev.download_body_forces(), table), i
            assert dev.download_body_forces().tobytes() == twin.download_body_forces().tobytes(), i
            assert _saved(dev) == _saved(twin), i
        dev.step(); twin.step()
        assert _state(dev) == _state(twin), i
        assert _counts(dev) == _counts(twin), i
    assert edits >= 6
    got = dev.download_body_forces()
    mirror = dev.scene.body_forces
    assert np.array_equal(got[mirror["body"].astype(np.int64)], mirror)


def test_state_files_round_trip_version_4_removes_the_table_and_nb_replay_replays():
    side = side_stream()
    s = _mixed(600, 44)
    g = nudge_b200.Sim(s, stream=side)
    rng = np.random.default_rng(9)
    g.set_body_forces(_random_entries(rng, np.arange(1, s.n_bodies, 2)))
    for _ in range(20):
        g.step()
    d = tempfile.mkdtemp(prefix="nb_body_force_state_")
    p1, p2, p4 = (os.path.join(d, x) for x in ("a.bin", "b.bin", "v4.bin"))
    g.save_state(p1)
    raw = open(p1, "rb").read()
    version, reserved = _header(raw)
    assert version == 5 and reserved[5] == 1 and reserved[4] == 0
    assert raw[-48 * s.n_bodies:] == g.download_body_forces().tobytes()
    h = nudge_b200.Sim(s, stream=side)
    h.load_state(p1)
    assert h.download_body_forces().tobytes() == g.download_body_forces().tobytes()
    for i in range(10):
        g.step(); h.step()
        assert _state(g) == _state(h), i
    # nb_replay prints the hash of every step's transforms
    exe = os.path.join(ROOT, "tools", "bin", "nb_replay")
    out = subprocess.run([exe, p1, "--steps", "10", "--iterations", str(int(s.iterations)), "--dump", p2], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stdout + out.stderr
    lines = [l.split() for l in out.stdout.strip().splitlines() if l.startswith("step")]
    h.load_state(p1)
    for i in range(10):
        h.step(); h.download_bodies()
        assert int(lines[i][lines[i].index("xf") + 1], 16) == fnv1a(h.transforms.tobytes()), i
    assert open(p2, "rb").read()[8:12] == struct.pack("<I", 5)
    # a version-4 file (kinematic set, no table) removes the table
    ks = s.copy(); ks.kinematic = np.array([(3, (0.0, 0.0, 0.0), (0.0, 0.0, 0.0), 0)], scenes.KINEMATIC)
    k = nudge_b200.Sim(ks, stream=side)
    k.save_state(p4)
    assert _header(open(p4, "rb").read())[0] == 4
    h.load_state(p4)
    assert np.array_equal(h.download_body_forces(), default_table(s.n_bodies))
    assert _header(_saved(h))[0] == 4


def test_upload_bodies_kinematic_bodies_and_shard_step():
    s = _mixed(300, 45)
    g = nudge_b200.Sim(s)
    rng = np.random.default_rng(10)
    ent = _random_entries(rng, np.arange(1, s.n_bodies))
    g.set_body_forces(ent)
    g.upload_bodies()   # the same count keeps the table
    assert np.array_equal(g.download_body_forces()[1:], ent)
    # a body made kinematic keeps its entry and ignores it
    k = 5
    ent5 = ent[ent["body"] == k].copy(); ent5["force"] = (0.0, 50.0, 0.0); ent5["gravity_scale"] = 2.0
    g.set_body_forces(ent5)
    g.upload_kinematic_bodies(np.array([(k, (0.0, 0.25, 0.0), (0.0, 0.0, 0.0), 0)], scenes.KINEMATIC))
    for _ in range(5):
        g.step_staged()
    g.download_bodies()
    assert g.momentum["velocity"][k].tolist() == [0.0, 0.25, 0.0]
    assert g.download_body_forces()[k].tobytes() == ent5[0].tobytes()
    assert _set(g, ent5) == NB_ERR_ARGUMENT   # a kinematic body's entry cannot be set
    g.upload_kinematic_bodies(None)
    # nb_shard_step refuses a context with a table
    b = nudge_b200.Sim(s)
    b.set_body_forces(ent[:4])
    b.shard_create(0, 1, None, 1, 1)
    with pytest.raises(nudge_b200.NudgeError, match="body force"):
        b.shard_step("peer")
    b.clear_body_forces()
    b.shard_step("peer")
    # another count drops the table
    g.reload(_mixed(298, 46))
    assert np.array_equal(g.download_body_forces(), default_table(299))
    assert _header(_saved(g))[0] == 1


def test_argument_errors_change_nothing():
    s = _mixed(300, 47)
    g = nudge_b200.Sim(s)
    rng = np.random.default_rng(11)
    g.upload_kinematic_bodies(np.array([(9, (0.0, 0.0, 0.0), (0.0, 0.0, 0.0), 0)], scenes.KINEMATIC))
    ent = _random_entries(rng, np.arange(10, 40))
    g.set_body_forces(ent)
    g.step_staged()
    want = g.download_body_forces()
    g.download_bodies(); idle = g.idle.copy()

    def bad(**kw):
        r = scenes.default_body_forces([20])
        for f, v in kw.items():
            r[f] = v
        return r
    cases = [scenes.default_body_forces([0]), scenes.default_body_forces([s.n_bodies]), scenes.default_body_forces([9]),
             scenes.default_body_forces([12, 13, 12]), bad(gravity_scale=np.inf), bad(linear_damping=np.nan), bad(force=(0.0, np.inf, 0.0)),
             bad(torque=(np.nan, 0.0, 0.0)), bad(angular_damping=-np.inf), bad(linear_damping=-0.5), bad(angular_damping=-1e-9), bad(flags=2),
             bad(flags=0x80000001)]
    for c in cases:
        good = scenes.default_body_forces([30]); good["gravity_scale"] = 3.0
        assert _set(g, np.concatenate([good, c])) == NB_ERR_ARGUMENT, c
    assert g.lib.nb_set_body_forces(g.ctx, None, 3, g.stream) == NB_ERR_ARGUMENT
    n = ctypes.c_uint32(0)
    small = np.zeros(s.n_bodies - 1, scenes.BODY_FORCE)
    assert g.lib.nb_download_body_forces(g.ctx, small.ctypes.data_as(ctypes.c_void_p), len(small), ctypes.byref(n), g.stream) == NB_ERR_CAPACITY
    assert n.value == s.n_bodies
    assert g.download_body_forces().tobytes() == want.tobytes()
    g.download_bodies()
    assert g.idle.tobytes() == idle.tobytes()
