"""Sensor colliders (nb_upload_sensors, DESIGN.md section 8.7) on the CPU: the restatement (tests/sensor_ref.py) without a table, and with an
all-zero one, is the unmodified oracle bit for bit over a run that sleeps and wakes; with sensors its physics is the filtered restatement with
the sensor colliders given category 0 and mask 0; its overlap lists follow their own BEGIN / END events while a pile sleeps inside a zone and
wakes again; Scene.copy and shard.local_scene carry the table, and nb_state_info reads the sensor state header."""
import ctypes, os
import numpy as np
import nudge_b200
from nudge_b200 import scenes, shard
from oracle import pyoracle
from tests.parity_util import stage_digests
from tests.filter_ref import FilteredOracleSim
from tests.sensor_ref import SensorOracleSim, add_sensors, masked_out, overlap_events
from tests.gpu_util import state_header

ZONES = [((0.0, -9.0, 0.0), (1.5, 1.5, 1.5)), ((2.5, -8.0, 1.0), (1.0, 2.5, 1.0)), ((-2.0, -7.0, -2.0), (2.0, 1.0, 2.0))]


def _base(seed=2):
    return scenes.demo_scene(80, 80, iterations=4, spread=2.5, height=12.0, seed=seed)


def _sensor_scene(seed=2):
    """Static zones just above the ground (its top is at y = -10), where the pile settles; sensor spheres around three bodies; two falling
    sensor spheres."""
    s = _base(seed)
    s.transforms["position"][1:, 1] -= 8.0
    return add_sensors(s, zones=ZONES, proximity=(3, 17, 40), falling=(5, 11))


def _sleep_then_wake(i, o):
    """Ahead of step i: at 20 every body falls asleep (one island: the whole pile sleeps), at 26 one body wakes it."""
    if i == 20:
        o.idle[:] = 0xff; o.momentum["velocity"][:] = 0; o.momentum["angular_velocity"][:] = 0
    if i == 26:
        o.idle[5] = 0


def test_restatement_without_a_table_and_with_an_all_zero_table_is_the_oracle():
    s = _base()
    la, da = stage_digests(pyoracle.OracleSim(s.copy()), True, 30, _sleep_then_wake)
    zero = s.copy(); zero.sensors = np.zeros(s.n_colliders, np.uint8)
    for scene in (s.copy(), zero):
        o = SensorOracleSim(scene)
        lb, db = stage_digests(o, True, 30, _sleep_then_wake)
        assert la == lb and np.array_equal(da, db)
        assert len(o.overlaps) == 0


def test_physics_equals_the_filtered_restatement_with_the_sensors_masked_out():
    s = _sensor_scene()
    o = SensorOracleSim(s)
    seen = []

    def before(i, x):
        if i:
            seen.append(len(x.overlaps))
        _sleep_then_wake(i, x)
    la, da = stage_digests(o, True, 30, before)
    lb, db = stage_digests(FilteredOracleSim(masked_out(s)), True, 30, _sleep_then_wake)
    assert la == lb and np.array_equal(da, db)
    assert max(seen) > 10                                     # the zones and the proximity spheres do overlap the pile


def test_overlaps_follow_their_events_while_the_pile_sleeps_inside_a_zone_and_wakes():
    s = _sensor_scene(seed=5)
    o = SensorOracleSim(s)
    prev = np.zeros(0, scenes.SENSOR_OVERLAP)
    asleep_overlaps = []
    n_begin = n_end = 0
    for i in range(40):
        _sleep_then_wake(i, o)
        o.step()
        cur = o.overlaps
        assert np.all(np.diff(cur["tags"].astype(np.float64)) > 0)           # one entry per pair, ascending
        ev = o.sensor_events(i)
        ends, begins = ev[ev["kind"] == scenes.SENSOR_END], ev[ev["kind"] == scenes.SENSOR_BEGIN]
        assert np.all(ev["kind"][:len(ends)] == scenes.SENSOR_END)          # ENDs first
        keys = set(prev["tags"].tolist()) - set(ends["tags"].tolist()) | set(begins["tags"].tolist())
        assert keys == set(cur["tags"].tolist()), i                         # overlaps(s) = overlaps(s-1) - END + BEGIN
        for e in begins:
            row = cur[cur["tags"] == e["tags"]][0]
            assert (e["body_a"], e["body_b"]) == (row["body_a"], row["body_b"])
        n_begin += len(begins); n_end += len(ends)
        if 20 <= i < 26:
            assert o.active.count == 0                                      # the pile sleeps ...
            asleep_overlaps.append(len(cur))
        prev = cur.copy()
    assert min(asleep_overlaps) > 0                                         # ... and keeps overlapping the zones
    assert n_begin > 0 and n_end > 0


def test_overlap_events_order_and_fields():
    old = np.zeros(3, scenes.SENSOR_OVERLAP); old["tags"] = (1 | 5 << 32, 2 | 5 << 32, 3 | 9 << 32); old["body_a"] = (1, 2, 3); old["body_b"] = 0
    cur = np.zeros(2, scenes.SENSOR_OVERLAP); cur["tags"] = (0 | 5 << 32, 2 | 5 << 32); cur["body_a"] = (7, 2); cur["body_b"] = (0, 0)
    ev = overlap_events(old, cur, 12)
    assert ev["kind"].tolist() == [scenes.SENSOR_END, scenes.SENSOR_END, scenes.SENSOR_BEGIN]
    assert ev["tags"].tolist() == [1 | 5 << 32, 3 | 9 << 32, 0 | 5 << 32]
    assert ev["body_a"].tolist() == [1, 3, 7] and set(ev["step"].tolist()) == {12}
    assert not ev["contacts"].any() and not ev["penetration"].any() and not ev["impulse"].any()


def test_scene_copy_and_shard_rows_carry_the_sensor_table():
    s = _sensor_scene()
    c = s.copy()
    assert np.array_equal(c.sensors, s.sensors) and c.sensors is not s.sensors
    assert scenes.Scene(1, 1, 0).sensors is None
    g = scenes.demo_scene(200, 200, iterations=4, spread=8.0, height=4.0, seed=5)
    g.sensors = (np.arange(g.n_colliders) % 3 == 0).astype(np.uint8)
    part = shard.partition(g, 2, margin=0.5)
    sens_of_tag = dict(zip(np.concatenate([g.box_tags, g.sphere_tags]).tolist(), g.sensors.tolist()))
    ghosts = 0
    for rank in range(2):
        loc, _ = shard.local_scene(g, part["owned"][rank], part["ghosts"][rank])
        assert loc.sensors.dtype == np.uint8 and len(loc.sensors) == loc.n_colliders
        assert loc.sensors.tolist() == [sens_of_tag[t] for t in np.concatenate([loc.box_tags, loc.sphere_tags]).tolist()]
        ghosts += len(part["ghosts"][rank])
    assert ghosts > 0
    loc, _ = shard.local_scene(_base(), [1, 2, 3], [])
    assert loc.sensors is None


def test_state_info_reads_the_sensor_header(tmp_path):
    lib = nudge_b200.load_library()
    counts = (ctypes.c_uint32 * 5)()
    for name, version, reserved, ok in (("v3", 3, (0, 0, 1, 4096) + (0,) * 4, True), ("v3f", 3, (1, 1, 1, 0) + (0,) * 4, True),
                                        ("v3bad", 3, (0, 0, 0, 4096) + (0,) * 4, False), ("v4", 4, (0, 0, 1, 0) + (0,) * 4, False),
                                        ("v4s", 4, (0, 0, 1, 4096, 1, 0, 0, 0), True), ("v4k", 4, (1, 1, 0, 0, 3, 0, 0, 0), True),
                                        ("v4s2", 4, (0, 0, 2, 0, 1, 0, 0, 0), False), ("v4k0", 4, (0, 0, 0, 0, 0, 0, 0, 0), False),
                                        ("v5", 5, (0, 0, 1, 0, 1, 0, 0, 0), False), ("v1r", 1, (7, 9, 2, 5, 0, 3, 3, 3), True),
                                        ("v2r", 2, (1, 1, 2, 0, 0, 0, 0, 0), True)):
        p = tmp_path / (name + ".bin")
        p.write_bytes(state_header(version, reserved))
        r = lib.nb_state_info(os.fsencode(str(p)), counts)
        assert (r == 0) == ok, name
        if ok:
            assert list(counts) == [1000, 600, 400, 7, 12345]


def test_the_bindings_export_the_sensor_calls():
    lib = nudge_b200.load_library()
    for f in ("nb_upload_sensors", "nb_download_sensor_overlaps"):
        assert f in nudge_b200.EXPORTS and hasattr(lib, f)
