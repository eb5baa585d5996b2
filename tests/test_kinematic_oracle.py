"""Kinematic bodies (nb_upload_kinematic_bodies, DESIGN.md section 8.8) on the CPU: the restatement (tests/kinematic_ref.py) without a set,
and with an empty one, is the unmodified oracle bit for bit over a run whose pile sleeps and wakes; with the ground moved onto a kinematic
body at rest it reproduces the UNMODIFIED REFERENCE on the original scene at every stage (the digests tests/golden/oracle_vs_ref.npz
recorded from it); and a moving platform carries its pile without ever changing its own velocity."""
import os
import numpy as np
from nudge_b200 import scenes
from oracle import pyoracle
from tests.parity_util import stage_digests
from tests.kinematic_ref import KinematicOracleSim, AsGround, with_kinematic_ground, two_kinematic_platforms, READ_ONLY

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "oracle_vs_ref.npz")


def _sleep_and_wake(rows):
    """Digests of every stage over a run in which most of a small pile is put to sleep and a falling body later wakes part of it."""
    s = scenes.demo_scene(120, 120, iterations=4, spread=6.0, height=6.0, seed=11)
    sleepy = np.random.default_rng(5).random(s.n_bodies) < 0.8
    seen = []

    def make(kind):
        o = pyoracle.OracleSim(s, contact_capacity=1 << 15) if kind == "oracle" else KinematicOracleSim(s, contact_capacity=1 << 15)
        if kind == "restated":
            o.upload_kinematic_bodies(rows)
        return o

    def before(i, sim):
        if i == 40:
            sim.idle[sleepy] = 0xff
            sim.momentum["velocity"][sleepy] = 0; sim.momentum["angular_velocity"][sleepy] = 0
        if i == 44:   # throw one awake body into the sleeping pile
            b = int(np.nonzero(~sleepy[1:])[0][0]) + 1
            sim.momentum["velocity"][b] = (0.0, -8.0, 0.0)
        if i > 40:
            seen.append(sim.contacts.sleeping_count)
    want = stage_digests(make("oracle"), True, 50, before)
    seen.clear()
    got = stage_digests(make("restated"), True, 50, before)
    assert max(seen) > 0, "the run never produced sleeping pairs"
    return want, got


def test_no_set_is_the_oracle_through_sleep_and_wake():
    (labels, want), (_, got) = _sleep_and_wake(None)
    bad = np.nonzero((want != got).any(axis=1))[0]
    assert not len(bad), "first differing stage: %s" % labels[bad[0]]


def test_empty_set_is_the_oracle_through_sleep_and_wake():
    (labels, want), (_, got) = _sleep_and_wake(np.zeros(0, scenes.KINEMATIC))
    bad = np.nonzero((want != got).any(axis=1))[0]
    assert not len(bad), "first differing stage: %s" % labels[bad[0]]


def _anchor(name, scene, steps):
    """The ground on a kinematic body at rest, viewed as the original scene, against the reference's recorded digests of that scene."""
    k_scene, k = with_kinematic_ground(scene)
    o = KinematicOracleSim(k_scene, contact_capacity=max(1024, 64 * scene.n_bodies))
    labels, got = stage_digests(AsGround(o, k), True, steps)
    want = np.load(GOLDEN)[name]
    assert got.shape == want.shape
    bad = np.nonzero((got != want).any(axis=1))[0]
    assert not len(bad), "%s: %d of %d stages differ from the reference, first: %s" % (name, len(bad), len(got), labels[bad[0]])


def test_kinematic_ground_at_rest_is_the_reference_small_mixed_scene():
    _anchor("small_mixed_scene_every_stage", scenes.demo_scene(100, 100, iterations=4, spread=2.0, height=20.0), 30)


def test_kinematic_ground_at_rest_is_the_reference_rotated_box_drop():
    _anchor("rotated_box_drop", scenes.box_drop(1500, iterations=8), 12)


def test_pairs_of_non_dynamic_bodies_with_a_kinematic_one_are_dropped():
    """A second ground collider on the kinematic body overlapping the first: no pair between them, while the same two colliders on body 0
    stay a (counted, contact-free) pair as in the reference."""
    s = scenes.demo_scene(20, 20, iterations=4, spread=2.0, height=4.0, seed=3)
    s.box_tags = np.concatenate([s.box_tags, [np.uint32(s.n_colliders)]])
    s.box_data = np.concatenate([s.box_data, s.box_data[:1]])
    s.box_transforms = np.concatenate([s.box_transforms, s.box_transforms[:1]])
    s.box_transforms["position"][-1, 0] = 50.0
    k_scene, k = with_kinematic_ground(s)
    plain = pyoracle.OracleSim(s, contact_capacity=1 << 14); plain.collide()
    o = KinematicOracleSim(k_scene, contact_capacity=1 << 14); o.collide()
    pv, kv = plain.pairs_view(), o.pairs_view()
    ground = {0, s.n_boxes - 1}
    both = lambda v: [(a, b) for a, b in zip(v["lo"].tolist(), v["hi"].tolist()) if a in ground and b in ground]
    assert len(both(pv)) == 1 and both(kv) == []
    assert len(kv["lo"]) == len(pv["lo"]) - 1


def test_rising_platform_carries_its_pile_and_keeps_its_velocity():
    base = scenes.box_drop(200, iterations=4, density_L=12.0, spacing=(2.2, 2.2, 2.2), rotate=False)
    k_scene, k = with_kinematic_ground(base)
    o = KinematicOracleSim(k_scene, contact_capacity=1 << 15)
    for _ in range(240):   # settle on the platform at rest
        o.step()
    o.upload_kinematic_bodies(np.array([(k, (0.0, 0.5, 0.0), (0.0, 0.0, 0.0), 0)], scenes.KINEMATIC))
    v0 = o.momentum[k].copy()
    y0 = float(o.transforms["position"][k, 1])
    for i in range(60):
        o.step()
        assert o.momentum[k]["velocity"].tolist() == v0["velocity"].tolist()
        assert o.momentum[k]["angular_velocity"].tolist() == v0["angular_velocity"].tolist()
        assert k in o.active_indices[:o.active.count].tolist()
    rise = float(o.transforms["position"][k, 1]) - y0
    assert abs(rise - 60 * float(base.time_step) * 0.5) < 1e-3
    c = o.constraints_view()
    assert ((c["a"] & READ_ONLY) != 0).any() or ((c["b"] & READ_ONLY) != 0).any()
    # the boxes resting on it rise with it: the lowest layer's mean vertical velocity is the platform's
    low = np.argsort(o.transforms["position"][1:k, 1])[:20] + 1
    assert abs(float(o.momentum["velocity"][low, 1].mean()) - 0.5) < 0.1


def test_pile_on_a_stopped_platform_sleeps_and_wakes_when_it_moves():
    base = scenes.box_drop(120, iterations=4, density_L=12.0, spacing=(2.2, 2.2, 2.2), rotate=False)
    k_scene, k = with_kinematic_ground(base)
    o = KinematicOracleSim(k_scene, contact_capacity=1 << 15)
    for _ in range(1200):
        o.step()
        if o.active.count == 0:
            break
    assert o.active.count == 0, "the pile never fell asleep"
    o.upload_kinematic_bodies(np.array([(k, (0.0, 0.0, 0.3), (0.0, 0.0, 0.0), 0)], scenes.KINEMATIC))
    o.collide()
    assert o.active.count > 1 and k in o.active_indices[:o.active.count].tolist()


def test_two_kinematic_bodies_pair_and_island_rules():
    """Two kinematic slabs overlapping each other and the ground (body 0), the pile asleep, K1 moving and K2 at rest.  Against the oracle's
    all-awake run of the same scene without a set: exactly the pairs of two non-dynamic bodies with a kinematic one are gone (the two ground
    colliders on body 0 would stay); the active bodies are K1 and every dynamic body that reaches K1 through contacts between dynamic bodies
    (a breadth-first walk, not a union-find), so the boxes that only touch K2 sleep."""
    s, k1, k2 = two_kinematic_platforms()
    plain = s.copy(); plain.kinematic = None
    a = pyoracle.OracleSim(plain, contact_capacity=1 << 16); a.collide()
    o = KinematicOracleSim(s, contact_capacity=1 << 16)
    o.upload_kinematic_bodies(np.array([(k1, (0.0, 0.1, 0.0), (0.0, 0.0, 0.0), 0), (k2, (0.0, 0.0, 0.0), (0.0, 0.0, 0.0), 0)], scenes.KINEMATIC))
    o.idle[1:k1] = 0xff
    o.collide()
    body = np.concatenate([s.box_transforms["body"], s.sphere_transforms["body"]]).astype(np.int64)
    pv, kv = a.pairs_view(), o.pairs_view()
    nondyn, kin = {0, k1, k2}, {k1, k2}
    drop = np.array([x in nondyn and y in nondyn and (x in kin or y in kin) for x, y in zip(body[pv["lo"]].tolist(), body[pv["hi"]].tolist())], bool)
    kinds = {(min(x, y), max(x, y)) for x, y in zip(body[pv["lo"]][drop].tolist(), body[pv["hi"]][drop].tolist())}
    assert kinds == {(0, k1), (0, k2), (k1, k2)}, kinds
    assert np.array_equal(kv["lo"], pv["lo"][~drop]) and np.array_equal(kv["hi"], pv["hi"][~drop])
    c = a.contacts_view()
    edges = {}
    for x, y in zip(c["bodies"]["a"].tolist(), c["bodies"]["b"].tolist()):
        edges.setdefault(x, set()).add(y); edges.setdefault(y, set()).add(x)
    seen, todo = set(), [b for b in edges.get(k1, ()) if b not in nondyn]
    while todo:
        b = todo.pop()
        if b in seen:
            continue
        seen.add(b)
        todo += [x for x in edges.get(b, ()) if x not in nondyn]
    want = sorted(seen | {k1})
    got = o.active_indices[:o.active.count].tolist()
    assert got == want and 10 < len(seen) < k1 - 11, (len(got), len(want))
    assert o.contacts.sleeping_count > 0
    # both at rest: everything sleeps; K2 moving instead: its side wakes
    o.upload_kinematic_bodies(np.array([(k1, (0.0, 0.0, 0.0), (0.0, 0.0, 0.0), 0), (k2, (0.0, 0.0, 0.0), (0.0, 0.0, 0.0), 0)], scenes.KINEMATIC))
    o.collide()
    assert o.active.count == 0
    o.upload_kinematic_bodies(np.array([(k1, (0.0, 0.0, 0.0), (0.0, 0.0, 0.0), 0), (k2, (0.0, 0.0, 0.0), (0.0, 0.3, 0.0), 0)], scenes.KINEMATIC))
    o.collide()
    got2 = set(o.active_indices[:o.active.count].tolist())
    assert k2 in got2 and k1 not in got2 and len(got2 - {k2}) > 10
