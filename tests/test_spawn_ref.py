"""The spawn / despawn restatement (tests/spawn_ref.py) on hand-built cases, and its wake set on the oracle: after a pile settles and sleeps,
removing its bottom box wakes exactly the bodies whose cache entries touched that box, and the next oracle collide activates their island and
no other.  CPU only."""
import numpy as np
from nudge_b200 import scenes
from tests.spawn_ref import REMOVED, add_bodies, rebuild_oracle, remove_bodies, live_scene
from tests.test_body_impulse_oracle import two_piles, settle_and_sleep


def _scene():
    """Bodies 0..5: body 0 carries the ground box and a sphere; body 2 a box and a sphere; body 3 no collider; bodies 1, 4, 5 one box each."""
    s = scenes.Scene(6, 5, 2)
    s.transforms["position"][:, 1] = np.arange(6, dtype=np.float32)
    s.momentum["velocity"][:, 0] = np.arange(6, dtype=np.float32)
    s.properties["mass_inverse"] = np.arange(6, dtype=np.float32)
    s.idle[:] = 0xff
    s.box_tags[:] = (10, 11, 12, 14, 15)
    s.box_transforms["body"] = (0, 1, 2, 4, 5)
    s.box_data["size"] = 0.5
    s.sphere_tags[:] = (20, 22)
    s.sphere_transforms["body"] = (0, 2)
    s.sphere_data["radius"] = 0.5
    s.connections = np.array([(1, 2), (0, 4), (3, 5), (2, 0)], scenes.PAIR32)
    s.collision_filters = np.zeros(7, scenes.FILTER); s.collision_filters["category"] = np.arange(7)
    s.sensors = np.array([0, 0, 1, 0, 0, 1, 0], np.uint8)
    s.kinematic = np.array([(5, (1, 0, 0), (0, 0, 0), 0), (3, (0, 0, 0), (0, 0, 0), 0)], scenes.KINEMATIC)
    return s


def _rows(pairs):
    from nudge_b200 import ROW
    r = np.zeros(len(pairs), ROW)
    r["a"] = [p[0] for p in pairs]; r["b"] = [p[1] for p in pairs]; r["impulse"] = np.arange(len(pairs), dtype=np.float32)
    return r


def test_removing_a_body_with_a_box_and_a_sphere():
    s = _scene()
    rows = _rows([(1, 2), (4, 0), (5, 1), (2, 2)])
    ov = np.array([(10 | 12 << 32, 0, 2), (11 | 15 << 32, 1, 5), (14 | 22 << 32, REMOVED, 2)], scenes.SENSOR_OVERLAP)
    cache = np.array([12 | 11 << 32, 14 | 22 << 32, 10 | 15 << 32], np.uint64)
    out, r, o, woken = remove_bodies(s, [2], cache, rows, ov)
    assert out.n_bodies == 5 and np.array_equal(out.transforms["position"][:, 1], [0, 1, 3, 4, 5])
    assert np.array_equal(out.properties["mass_inverse"], [0, 1, 3, 4, 5])
    assert np.array_equal(out.box_tags, [10, 11, 14, 15]) and np.array_equal(out.box_transforms["body"], [0, 1, 3, 4])
    assert np.array_equal(out.sphere_tags, [20]) and np.array_equal(out.sphere_transforms["body"], [0])
    assert np.array_equal(out.collision_filters["category"], [0, 1, 3, 4, 5]) and np.array_equal(out.sensors, [0, 0, 0, 0, 1])
    assert out.connections.tolist() == [(0, 3), (2, 4)]
    assert sorted(out.kinematic["body"].tolist()) == [2, 4]
    assert r[["a", "b"]].tolist() == [(3, 0), (4, 1)] and r["impulse"].tolist() == [1.0, 2.0]
    assert o[["body_a", "body_b"]].tolist() == [(0, REMOVED), (1, 4), (REMOVED, REMOVED)]
    # woken: body 1 (cache pair 12-11 and the connection 1-2), body 4 (cache pair 14-22); never body 0
    assert np.nonzero(woken)[0].tolist() == [1, 4]
    assert out.idle.tolist() == [0xff, 0, 0xff, 0, 0xff]


def test_removing_a_body_without_a_collider_and_keeping_body_0s_colliders():
    s = _scene()
    s.kinematic = None
    out, _, _, woken = remove_bodies(s, [3], np.zeros(0, np.uint64))
    assert np.array_equal(out.box_tags, s.box_tags) and np.array_equal(out.sphere_tags, s.sphere_tags)
    assert np.array_equal(out.box_transforms["body"], [0, 1, 2, 3, 4]) and np.array_equal(out.sphere_transforms["body"], [0, 2])
    assert out.connections.tolist() == [(1, 2), (0, 3), (2, 0)]
    assert np.nonzero(woken)[0].tolist() == [5]   # the connection 3-5 (old indices); body 5 becomes 4
    assert out.idle[4] == 0


def test_removing_every_dynamic_body_leaves_the_world():
    s = _scene()
    rows = _rows([(1, 0), (0, 4)])
    out, r, _, _ = remove_bodies(s, [5, 1, 3, 2, 4], None, rows)
    assert out.n_bodies == 1 and out.kinematic is None and len(r) == 0 and len(out.connections) == 0
    assert np.array_equal(out.box_tags, [10]) and np.array_equal(out.sphere_tags, [20])
    assert (out.box_transforms["body"] == 0).all() and (out.sphere_transforms["body"] == 0).all()


def test_adding_a_fragment_inserts_table_entries_in_collider_order():
    s = _scene()
    fr = scenes.fragment([(0, 1, 0), (0, 3, 0)], "box", first_tag=30)
    sp = scenes.fragment([(1, 1, 0)], "sphere", first_tag=40)
    both = scenes.Scene(0, 0, 0)
    for k in ("transforms", "properties", "momentum", "idle"):
        setattr(both, k, np.concatenate([getattr(fr, k), getattr(sp, k)]))
    both.box_tags, both.box_data, both.box_transforms = fr.box_tags, fr.box_data, fr.box_transforms
    sx = sp.sphere_transforms.copy(); sx["body"] += 2
    both.sphere_tags, both.sphere_data, both.sphere_transforms = sp.sphere_tags, sp.sphere_data, sx
    both.collision_filters = np.zeros(3, scenes.FILTER); both.collision_filters["category"] = (100, 101, 102)
    both.sensors = np.array([1, 0, 1], np.uint8)
    out = add_bodies(s, both)
    assert out.n_bodies == 9 and np.array_equal(out.box_transforms["body"][5:], [6, 7]) and out.sphere_transforms["body"][2] == 8
    assert out.collision_filters["category"].tolist() == [0, 1, 2, 3, 4, 100, 101, 5, 6, 102]
    assert out.sensors.tolist() == [0, 0, 1, 0, 0, 1, 0, 1, 0, 1]
    assert out.properties["mass_inverse"][6] == np.float32(1.0) / np.float32(8.0 * 0.125)


def test_wake_set_on_the_oracle_is_the_removed_boxs_cache_partners_and_wakes_only_its_island():
    from oracle import pyoracle
    s, pile_a, pile_b = two_piles()
    o = pyoracle.OracleSim(s)
    settle_and_sleep(o)
    o.step()   # the cache now holds the culled entries of the sleeping pairs
    assert o.cache.count > 0 and (o.idle[1:] == 0xff).all()
    bottom = int(pile_a[0])
    tag = int(s.box_tags[list(s.box_transforms["body"]).index(bottom)])
    keys = o.cache_tags[:o.cache.count]
    partners = set()
    for k in keys.tolist():
        a, b = k & 0xffffffff, k >> 32
        if tag in (a, b):
            t = b if a == tag else a
            partners.update(int(x) for x in np.concatenate([s.box_transforms["body"][s.box_tags == t], s.sphere_transforms["body"][s.sphere_tags == t]]))
    partners.discard(0)
    assert partners == {int(pile_a[1])}
    out, _, _, woken = remove_bodies(live_scene(o), [bottom], keys)
    assert set(np.nonzero(woken)[0].tolist()) == partners
    o2 = rebuild_oracle(o, out)
    o2.collide()
    moved = lambda b: int(b) - (1 if b > bottom else 0)
    want = sorted(moved(b) for b in pile_a if b != bottom)
    assert sorted(o2.contacts_view()["active"].tolist()) == want
    assert (o2.idle[[moved(b) for b in pile_b]] == 0xff).all()
