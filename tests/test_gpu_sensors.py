"""Sensor colliders on the device (nb_upload_sensors, DESIGN.md section 8.7): a sensor context against the same scene with the sensor
colliders filtered out (category 0, mask 0), bit for bit at every step; the overlap lists and sensor events against the restatement
(tests/sensor_ref.py) through sleep and wake; the same decision as the contacts on the reference-recorded edge-case geometry; graph replay
while the table changes; launch counts, throughput mode, capacity overflow, state files with nb_replay, and the argument errors."""
import ctypes, os, struct, subprocess, tempfile
import numpy as np
import pytest
import nudge_b200
from nudge_b200 import scenes
from tests import np_edge_cases as E
from tests.sensor_ref import SensorOracleSim, add_sensors, masked_out
from tests.gpu_util import fnv1a, side_stream

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "np_edge_cases.npz")
NB_ERR_ARGUMENT, NB_ERR_OVERFLOW = -3, -4
SENSOR_KINDS = (scenes.SENSOR_BEGIN, scenes.SENSOR_END)


def _pile():
    """The 8,191-box pile with 36 static zones on the ground and sensor spheres around 40 of its boxes."""
    s = scenes.box_drop(8191, iterations=8)
    zones = [((x, 1.5, z), (1.5, 1.5, 1.5)) for x in np.linspace(-12.0, 12.0, 6) for z in np.linspace(-12.0, 12.0, 6)]
    return add_sensors(s, zones=zones, proximity=np.arange(1, 8191, 200))


def _mixed(seed=21):
    """Boxes and spheres on the ground through static zones, sensor spheres around a few bodies, a few falling sensor spheres."""
    s = scenes.demo_scene(300, 300, iterations=4, spread=4.0, height=14.0, seed=seed)
    s.transforms["position"][1:, 1] -= 9.0
    zones = [((x, -8.5, z), (1.2, 1.5, 1.2)) for x in (-2.5, 0.0, 2.5) for z in (-2.5, 2.5)]
    return add_sensors(s, zones=zones, proximity=(4, 50, 333, 420), falling=(7, 77, 177))


def _sleep_host(x, on):
    """Every body asleep and at rest (the pile is one island), or body 5 woken."""
    if on:
        x.idle[:] = 0xff; x.momentum["velocity"][:] = 0; x.momentum["angular_velocity"][:] = 0
    else:
        x.idle[5] = 0


def _sleep(x, on):
    x.download_bodies(); _sleep_host(x, on); x.upload_bodies()


def _state(x):
    x.download_bodies(); x.download_contacts(); x.download_cache()
    c = x.contacts_view()
    parts = [x.transforms, x.momentum, x.idle, c["data"], c["bodies"], c["tags"], c["features"], c["sleeping"], c["active"]]
    cv = x.cache_view()
    return b"".join(np.ascontiguousarray(a).tobytes() for a in parts + [cv["tags"], cv["features"], cv["data"]])


@pytest.mark.parametrize("which", ["pile_8191", "mixed"])
def test_sensors_change_no_physics_bit_for_bit_at_every_step(which):
    s = _pile() if which == "pile_8191" else _mixed()
    steps, sleep_at = (160, 120) if which == "pile_8191" else (80, 50)
    a = nudge_b200.Sim(s, stream=side_stream()); b = nudge_b200.Sim(masked_out(s), stream=side_stream())
    for x in (a, b):
        x.enable_contact_events(1 << 18)
    overlapped = sensor_events = 0
    for i in range(steps):
        if i in (sleep_at, sleep_at + 6):
            for x in (a, b):
                _sleep(x, i == sleep_at)
        a.step(); b.step()
        assert _state(a) == _state(b), "%s step %d" % (which, i)
        ea, da = a.contact_events(); eb, db = b.contact_events()
        assert da == db == 0
        sens = np.isin(ea["kind"], SENSOR_KINDS)
        assert ea[~sens].tobytes() == eb.tobytes(), "%s step %d: contact events" % (which, i)
        assert not sens.any() or sens[np.argmax(sens):].all()          # the sensor events come after the contact events
        sensor_events += int(sens.sum())
        overlapped = max(overlapped, len(a.sensor_overlaps()))
        assert a.counts().overflow == 0
    print("%s: up to %d overlaps, %d sensor events" % (which, overlapped, sensor_events))
    assert overlapped > 30 and sensor_events > 30


def test_overlaps_and_sensor_events_equal_the_restatement_through_sleep_and_wake():
    from oracle import events_ref
    s = _mixed(seed=22)
    o = SensorOracleSim(s, contact_capacity=1 << 17); rec = events_ref.OracleEvents(o)   # the all-awake oracle run holds every pair's contacts
    g = nudge_b200.Sim(s, contact_capacity=o.cap, stream=side_stream())
    g.enable_contact_events(1 << 16)
    asleep = []
    for i in range(70):
        if i in (45, 52):
            _sleep_host(o, i == 45); _sleep(g, i == 45)
        want = np.concatenate([rec.step(), o.sensor_events(i)])
        g.step()
        got, dropped = g.contact_events()
        assert dropped == 0 and got.tobytes() == want.tobytes(), "step %d: %d vs %d events" % (i, len(got), len(want))
        ov = g.sensor_overlaps()
        assert ov.tobytes() == o.overlaps.tobytes(), "step %d: %d vs %d overlaps" % (i, len(ov), len(o.overlaps))
        if 45 <= i < 52:
            assert g.counts().active == 0
            asleep.append(len(ov))
    assert min(asleep) > 0


def test_same_decision_as_the_contacts_on_the_edge_case_geometry():
    golden = np.load(GOLDEN)
    total = hits = 0
    for es in E.all_scenes():
        s = es.scene.copy()
        ncol = s.n_colliders
        first = {}
        for i, c in enumerate(es.col_cluster.tolist()):   # one collider of every cluster becomes the sensor
            first.setdefault(c, i)
        s.sensors = np.zeros(ncol, np.uint8); s.sensors[list(first.values())] = 1
        want_g = E.golden_of(golden, es)
        tags = np.concatenate([s.box_tags, s.sphere_tags]).astype(np.uint64)
        ta = (want_g["tags"] >> np.uint64(32)) & np.uint64(0xffff); tb = want_g["tags"] >> np.uint64(48)
        sensor_tags = set(tags[s.sensors != 0].tolist())
        want = set()
        for x, y in zip(ta.tolist(), tb.tolist()):
            if (x in sensor_tags) != (y in sensor_tags):
                want.add(min(x, y) | max(x, y) << 32)
        g = nudge_b200.Sim(s, contact_capacity=max(1024, 16 * ncol), debug=True)
        g.collide()
        assert g.counts().overflow == 0
        got = g.sensor_overlaps()
        assert len(set(got["tags"].tolist())) == len(got)
        if set(got["tags"].tolist()) != want:
            cl = es.cluster_of_tag()
            bad = sorted(set(got["tags"].tolist()) ^ want)
            raise AssertionError("%s: %d overlaps, %d expected; first difference: %s" % (es.name, len(got), len(want), es.describe(cl[bad[0] & 0xffffffff])))
        total += len(first); hits += len(want)
    print("edge cases: %d clusters with a sensor, %d overlapping" % (total, hits))
    assert hits > 100 and total > hits


def test_graph_replay_equals_the_stage_calls_while_the_table_changes():
    s = _mixed(seed=23)
    table = s.sensors
    s.sensors = None
    other = table.copy(); other[::5] = 1 - other[::5]
    # without the table the zones and sensor spheres are solid colliders inside the starting pile: room for the pairs and contacts that makes
    a, b = (nudge_b200.Sim(s, stream=side_stream(), pair_capacity=1 << 16, contact_capacity=1 << 17) for _ in range(2))
    for x in (a, b):
        x.enable_contact_events(1 << 16)
    for i in range(40):
        if i in (10, 20, 30):
            f = {10: table, 20: other, 30: None}[i]
            a.upload_sensors(f); b.upload_sensors(f)
        a.step(); b.step_staged()
        assert a.counts().overflow == 0 and _state(a) == _state(b), i
        assert a.sensor_overlaps().tobytes() == b.sensor_overlaps().tobytes(), i
        ea, _ = a.contact_events(); eb, _ = b.contact_events()
        assert ea.tobytes() == eb.tobytes(), i
        if 10 <= i < 30:
            assert len(a.sensor_overlaps()) > 0
    assert a.debug_scalar("graph_active") == 1


def test_launch_counts_and_throughput_mode():
    s = _mixed(seed=24)
    plain = nudge_b200.Sim(masked_out(s), stream=side_stream())
    plain.upload_collision_filters(None)
    nosens = nudge_b200.Sim(scenes.demo_scene(300, 300, iterations=4, spread=4.0, height=14.0, seed=24), stream=side_stream())
    sens = nudge_b200.Sim(s, stream=side_stream())
    zero = nudge_b200.Sim(s, stream=side_stream()); zero.upload_sensors(np.zeros(s.n_colliders, np.uint8))
    removed = nudge_b200.Sim(s, stream=side_stream()); removed.upload_sensors(None)
    used = {}
    for name, x in (("none", nosens), ("plain", plain), ("sensors", sens), ("zero", zero), ("removed", removed)):
        for i in range(3):
            before = x.launch_count()
            x.step() if i else x.step_staged()
            used.setdefault(name, []).append(x.launch_count() - before)
    assert used["none"][1:] == [61, 61] and used["plain"] == used["none"] and used["removed"] == used["none"], used   # [0]: the stage calls
    assert used["sensors"] == used["zero"] == [n + 6 for n in used["none"]], used
    p = nudge_b200.Sim(s); t = nudge_b200.Sim(s)
    t.set_solver_mode("throughput")
    for _ in range(30):
        p.step_staged()
    p.download_bodies()
    t.transforms[:] = p.transforms; t.momentum[:] = p.momentum; t.idle[:] = p.idle
    t.upload_bodies()
    p.collide(); t.collide()
    assert len(p.sensor_overlaps()) > 0 and p.sensor_overlaps().tobytes() == t.sensor_overlaps().tobytes()


def test_wrong_count_collider_change_and_overflow():
    s = _mixed(seed=25)
    g = nudge_b200.Sim(s)
    n = s.n_colliders
    f = np.ascontiguousarray(s.sensors)
    for bad in (n - 1, n + 1):
        assert g.lib.nb_upload_sensors(g.ctx, f.ctypes.data_as(ctypes.c_void_p), bad, 0, g.stream) == NB_ERR_ARGUMENT
    for _ in range(20):
        g.step_staged()
    assert len(g.sensor_overlaps()) > 0
    g._ck(g.lib.nb_upload_colliders(g.ctx, ctypes.byref(g.colliders), g.stream), "nb_upload_colliders")   # same count: kept
    g.collide(); assert len(g.sensor_overlaps()) > 0
    plain = scenes.demo_scene(300, 299, iterations=4, spread=4.0, height=14.0, seed=25)
    g.reload(plain)                                                                                         # another count: removed
    g.collide(); assert len(g.sensor_overlaps()) == 0
    assert g.lib.nb_upload_sensors(g.ctx, f.ctypes.data_as(ctypes.c_void_p), n, 0, g.stream) == NB_ERR_ARGUMENT
    # a too-small candidate capacity: the overflow bit, NB_ERR_OVERFLOW with a message that names it, no fault, and a clean step after
    h = nudge_b200.Sim(s)
    for _ in range(20):
        h.step_staged()
    h.upload_sensors(s.sensors, max_pairs=4)
    h.step_staged()
    c = nudge_b200.Counts()
    assert h.lib.nb_download_counts(h.ctx, ctypes.byref(c), h.stream) == NB_ERR_OVERFLOW
    assert c.overflow & 32 and "sensor" in h.lib.nb_last_error(h.ctx).decode()
    h.upload_sensors(s.sensors)
    h.step_staged()
    assert h.counts().overflow == 0 and len(h.sensor_overlaps()) > 0


def test_state_files_carry_the_table_and_replay():
    side = side_stream()
    s = _mixed(seed=26)
    g = nudge_b200.Sim(s, stream=side)
    for _ in range(25):
        g.step()
    d = tempfile.mkdtemp(prefix="nb_sensor_state_")
    p1, p2, p3 = (os.path.join(d, x) for x in ("a.bin", "b.bin", "plain.bin"))
    g.save_state(p1)
    raw = open(p1, "rb").read()
    version, = struct.unpack_from("<I", raw, 8); reserved = struct.unpack_from("<8I", raw, 36)
    assert version == 3 and reserved[2] == 1 and reserved[3] > 0
    k = s.n_colliders
    assert raw[len(raw) - (k + 15) // 16 * 16:][:k] == (s.sensors != 0).astype(np.uint8).tobytes()
    h = nudge_b200.Sim(_mixed(seed=99), stream=side)   # the same sizes, another state
    h.load_state(p1)
    for x in (g, h):
        x.enable_contact_events(1 << 16)
    for i in range(10):
        g.step(); h.step()
        eg, _ = g.contact_events(); eh, _ = h.contact_events()
        if i == 0:   # the load emptied the old overlaps: every overlap begins; g only begins the new ones
            assert (eh["kind"] == scenes.SENSOR_BEGIN).sum() == len(h.sensor_overlaps()) > 0
        else:
            assert eg.tobytes() == eh.tobytes()
    assert _state(g) == _state(h) and g.sensor_overlaps().tobytes() == h.sensor_overlaps().tobytes()
    exe = os.path.join(ROOT, "tools", "bin", "nb_replay")
    out = subprocess.run([exe, p1, "--steps", "10", "--iterations", str(int(s.iterations)), "--dump", p2], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stdout + out.stderr
    last = out.stdout.strip().splitlines()[-1].split()
    h.load_state(p1)
    for _ in range(10):
        h.step()
    h.download_bodies()
    assert int(last[last.index("xf") + 1], 16) == fnv1a(h.transforms.tobytes())
    assert open(p2, "rb").read()[8:12] == struct.pack("<I", 3)
    plain = nudge_b200.Sim(scenes.demo_scene(120, 120, iterations=4, seed=3), stream=side)
    plain.save_state(p3)
    assert struct.unpack_from("<I", open(p3, "rb").read(), 8)[0] == 1       # no sensors: version 1 as before
    h.load_state(p3)
    h.collide()
    assert len(h.sensor_overlaps()) == 0


def test_sharded_step_refuses_a_context_with_sensors():
    s = _mixed(seed=27)
    b = nudge_b200.Sim(s)
    b.shard_create(0, 1, None, 1, 1)
    with pytest.raises(nudge_b200.NudgeError, match="sensor"):
        b.shard_step("peer")
    b.upload_sensors(None)
    b.shard_step("peer")
