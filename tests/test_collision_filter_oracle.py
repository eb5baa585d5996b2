"""Collision filters (nb_upload_collision_filters, DESIGN.md section 8.6) on the CPU: the filtered restatement (tests/filter_ref.py) without a
table, and with an all-pass table, is the unmodified oracle bit for bit over a run with sleeping and waking islands; its pair list is the
oracle's minus the pairs the category / mask rule or the connected opt-out rejects, and its contacts only join passing colliders; a
sharded local scene carries the filter rows of its colliders, Scene.copy keeps them, and nb_state_info reads version-1 and 2 headers."""
import ctypes, os
import numpy as np
import nudge_b200
from nudge_b200 import scenes, shard
from oracle import pyoracle
from tests.parity_util import stage_digests
from tests.filter_ref import FilteredOracleSim
from tests.gpu_util import state_header


def _scene():
    return scenes.demo_scene(150, 150, iterations=4, spread=3.0, height=20.0, seed=7)


def _random_filters(n, seed=3):
    rng = np.random.default_rng(seed)
    f = np.zeros(n, scenes.FILTER)
    f["category"] = 1 << rng.integers(0, 3, n)                     # three categories
    f["mask"] = rng.integers(1, 8, n)                               # any non-empty subset of them
    return f


def _pairs(o):
    v = o.pairs_view()
    return v["lo"].astype(np.uint64) | (v["hi"].astype(np.uint64) << np.uint64(32)), v["lo"], v["hi"]


def _collide_pairs(scene, filters=None, flags=0):
    o = FilteredOracleSim(scene, contact_capacity=1 << 16)
    o.upload_collision_filters(filters, flags)
    o.collide()
    return _pairs(o), o


def test_filtered_pairs_are_the_unfiltered_pairs_that_pass_the_rule():
    s = _scene()
    (all_keys, lo, hi), _ = _collide_pairs(s)
    assert len(all_keys) > 500
    f = _random_filters(s.n_colliders)
    (keys, _, _), o = _collide_pairs(s, f)
    cat, mask = f["category"], f["mask"]
    keep = ((cat[lo] & mask[hi]) != 0) & ((cat[hi] & mask[lo]) != 0)
    assert 0 < keep.sum() < len(keep)
    assert np.array_equal(keys, all_keys[keep])                    # same order: the sorted list with the rejected pairs taken out
    c = o.contacts_view()
    col_of_tag = {int(t): i for i, t in enumerate(np.concatenate([s.box_tags, s.sphere_tags]))}
    for t in np.unique(c["tags"]):
        a, b = col_of_tag[int(t) & 0xffffffff], col_of_tag[int(t) >> 32]
        assert (cat[a] & mask[b]) and (cat[b] & mask[a])


def test_connected_opt_out_removes_the_pairs_of_connected_bodies():
    s = _scene()
    s.transforms["position"][1:7, 1] = -9.8                          # a few bodies on the ground (body 0, top at y = -10)
    body = np.concatenate([s.box_transforms["body"], s.sphere_transforms["body"]]).astype(np.int64)
    (all_keys, lo, hi), _ = _collide_pairs(s)
    ba, bb = body[lo], body[hi]
    touching = np.nonzero(ba != bb)[0]
    pick = touching[::3]                                            # connect the bodies of every third overlapping pair, some with body 0
    conn = np.unique(np.stack([np.minimum(ba[pick], bb[pick]), np.maximum(ba[pick], bb[pick])], 1), axis=0)
    conn[::2] = conn[::2, ::-1]                                     # either order
    s.connections = np.zeros(len(conn), scenes.PAIR32); s.connections["a"] = conn[:, 0]; s.connections["b"] = conn[:, 1]
    assert (conn == 0).any()
    (same, _, _), _ = _collide_pairs(s)                             # connections alone change no pair
    assert np.array_equal(same, all_keys)
    (keys, _, _), _ = _collide_pairs(s, None, scenes.FILTER_SKIP_CONNECTED)
    joined = set(map(tuple, np.sort(conn, 1).tolist()))
    keep = np.array([(min(x, y), max(x, y)) not in joined for x, y in zip(ba, bb)])
    assert 0 < keep.sum() < len(keep)
    assert np.array_equal(keys, all_keys[keep])
    f = _random_filters(s.n_colliders, seed=9)                      # both rules together
    (keys, _, _), _ = _collide_pairs(s, f, scenes.FILTER_SKIP_CONNECTED)
    cat, mask = f["category"], f["mask"]
    keep &= ((cat[lo] & mask[hi]) != 0) & ((cat[hi] & mask[lo]) != 0)
    assert np.array_equal(keys, all_keys[keep])


def _sleep_then_wake(i, o):
    """Ahead of step i: at 20 every body falls asleep (one island: the whole pile sleeps), at 24 one body wakes it."""
    if i == 20:
        o.idle[:] = 0xff; o.momentum["velocity"][:] = 0; o.momentum["angular_velocity"][:] = 0
    if i == 24:
        o.idle[5] = 0


def test_restatement_without_filters_and_with_an_all_pass_table_is_the_oracle():
    s = scenes.demo_scene(80, 80, iterations=4, spread=2.0, height=15.0, seed=2)
    s.connections = np.zeros(4, scenes.PAIR32); s.connections["a"] = (1, 7, 30, 0); s.connections["b"] = (2, 8, 31, 40)
    la, da = stage_digests(pyoracle.OracleSim(s.copy()), True, 30, _sleep_then_wake)
    t = s.copy()
    t.collision_filters = np.zeros(s.n_colliders, scenes.FILTER); t.collision_filters["category"] = 0xffff; t.collision_filters["mask"] = 0xffff
    for scene in (s.copy(), t):
        o = FilteredOracleSim(scene)
        sleeping = []

        def before(i, x):
            sleeping.append(x.contacts.sleeping_count)
            _sleep_then_wake(i, x)
        lb, db = stage_digests(o, True, 30, before)
        assert la == lb and np.array_equal(da, db)
        assert max(sleeping) > 0 and sleeping[-1] == 0            # the pile slept, and woke again


def test_scene_copy_keeps_the_filters():
    s = _scene()
    s.collision_filters = _random_filters(s.n_colliders); s.filter_flags = scenes.FILTER_SKIP_CONNECTED
    c = s.copy()
    assert c.filter_flags == 1 and np.array_equal(c.collision_filters, s.collision_filters)
    assert c.collision_filters is not s.collision_filters
    assert scenes.Scene(1, 1, 0).collision_filters is None


def test_shard_local_scene_carries_the_filter_rows_of_its_colliders():
    s = scenes.demo_scene(200, 200, iterations=4, spread=8.0, height=4.0, seed=5)
    n = s.n_colliders
    s.collision_filters = np.zeros(n, scenes.FILTER)
    s.collision_filters["category"] = np.arange(n) % 65535 + 1     # unique per collider: the row identifies the collider
    s.collision_filters["mask"] = np.arange(n)[::-1] % 65535 + 1
    s.filter_flags = scenes.FILTER_SKIP_CONNECTED
    part = shard.partition(s, 2, margin=0.5)
    filt_of_tag = dict(zip(np.concatenate([s.box_tags, s.sphere_tags]).tolist(), s.collision_filters.tolist()))
    seen = 0
    for rank in range(2):
        loc, gids = shard.local_scene(s, part["owned"][rank], part["ghosts"][rank])
        assert loc.filter_flags == scenes.FILTER_SKIP_CONNECTED
        assert loc.collision_filters.dtype == scenes.FILTER and len(loc.collision_filters) == loc.n_colliders
        tags = np.concatenate([loc.box_tags, loc.sphere_tags]).tolist()
        assert loc.collision_filters.tolist() == [filt_of_tag[t] for t in tags]
        seen += len(part["ghosts"][rank])
    assert seen > 0                                                 # ghosts exist, and they kept their global rows


def test_state_info_reads_version_1_and_version_2_headers(tmp_path):
    lib = nudge_b200.load_library()
    counts = (ctypes.c_uint32 * 5)()
    for version, reserved in ((1, (0,) * 8), (2, (1, 1) + (0,) * 6), (2, (0, 1) + (0,) * 6)):
        p = tmp_path / ("v%d_%d.bin" % (version, reserved[0]))
        p.write_bytes(state_header(version, reserved))
        assert lib.nb_state_info(os.fsencode(str(p)), counts) == 0
        assert list(counts) == [1000, 600, 400, 7, 12345]
    p = tmp_path / "v3.bin"
    p.write_bytes(state_header(3))
    assert lib.nb_state_info(os.fsencode(str(p)), counts) != 0
