"""Pins the widened CPU restatement (oracle/nudge_oracle.cpp) against the UNMODIFIED reference on scenes whose collider tags are not the
generators' dense 0..K-1: permuted, sparse up to 0xFFFF, shared by several colliders, and with custom contacts appended after collide
(tags no collider carries, arbitrary feature words), bit for bit at every stage.  The reference's digests are stored in
tests/golden/tag_cases.npz, recorded by tests/golden/make_tag_golden.py.  Also checks the premises of the retagging helpers
(tests/tag_cases.py).  CPU only."""
import os
import numpy as np
import pytest
from nudge_b200 import scenes
from tests import tag_cases as T
from tests.parity_util import stage_digests

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "tag_cases.npz")
HIGH16 = (0xffff, 0xfff0, 0xc000, 0x8001)   # custom-contact tags beyond the collider range of the dense scenes


def _cap(s):
    return max(1024, 64 * s.n_bodies)


def _pile():
    return scenes.demo_scene(100, 100, iterations=4, spread=2.0, height=20.0)


def _sleepy_scene():
    return scenes.demo_scene(120, 120, iterations=4, spread=6.0, height=6.0, seed=11)


def _custom_hook(high, seed, append):
    def hook(i, sim):
        append(sim, T.custom_contacts(sim, i, high, seed))
    return hook


def _run(scene, steps, sleep_at=None, high=None, seed=0, seen=None):
    """A case: (make, wide) -> (labels, digests).  sleep_at: force all bodies but 1..10 asleep ahead of that step; high: append custom
    contacts with these tags after every collide."""
    sleepy = np.arange(scene.n_bodies) > 10   # all but ten bodies: most islands stay asleep whatever the trajectory

    def before(i, sim):
        if i == sleep_at:
            sim.idle[sleepy] = 0xff
            sim.momentum["velocity"][sleepy] = 0; sim.momentum["angular_velocity"][sleepy] = 0
        if seen is not None and i:
            seen.append((sim.contacts.sleeping_count, len(sim.impulses_view()["culled_tags"])))

    def case(make, wide):
        after = _custom_hook(high, seed, T.append_wide if wide else T.append_ref) if high is not None else None
        return stage_digests(make(scene, _cap(scene)), wide, steps, before if sleep_at is not None or seen is not None else None, after_collide=after)
    case.scene, case.steps, case.sleep_at, case.high, case.seed = scene, steps, sleep_at, high, seed
    return case


CASES = {
    "permuted_pile": _run(T.permuted(_pile(), seed=3)[0], 20),
    "sparse_monotone_16_pile": _run(T.monotone(_pile(), 16, seed=4)[0], 20),
    "shared_compound_pile": _run(T.shared(T.compound(_pile(), np.arange(1, 101, 3))), 20),
    "permuted_sleeping_islands": _run(T.permuted(_sleepy_scene(), seed=9)[0], 47, sleep_at=40),
    "dense_pile_custom_contacts": _run(_pile(), 12, high=HIGH16, seed=6),
    "permuted_sleeping_custom_contacts": _run(T.permuted(_sleepy_scene(), seed=7, max_tag=0xfff0)[0], 47, sleep_at=40, high=(0xffff, 0xfffe, 0xfff8), seed=8),
}


def _oracle(scene, cap):
    from oracle import pyoracle
    return pyoracle.OracleSim(scene, contact_capacity=cap)


@pytest.mark.parametrize("name", sorted(CASES))
def test_oracle_equals_reference_with_application_tags(name):
    want = np.load(GOLDEN)[name]
    labels, got = CASES[name](_oracle, True)
    assert got.shape == want.shape, "%s: %d stage digests, the reference recorded %d" % (name, len(got), len(want))
    bad = np.nonzero((got != want).any(axis=1))[0]
    assert not len(bad), "%s: %d of %d stages differ from the reference, first: %s" % (name, len(bad), len(got), labels[bad[0]])


def test_layout_rule_covers_every_width():
    assert [T.layout(b) for b in (1, 2)] == ["packed"] * 2
    assert all(T.layout(b) == "spread" for b in range(3, 24))
    assert T.layout(24) == "packed" and T.key_bits(24) == (64,)
    assert T.key_bits(23) == (63,) and T.key_bits(22) == (61,)
    assert all(T.layout(b) == "two-pass" for b in range(25, 33)) and T.key_bits(32) == (32, 64)
    assert all(T.layout(b, internal=False) == "two-pass" for b in range(1, 33))
    assert T.bits_for(2) == 1 and T.bits_for(3) == 2 and T.bits_for(1 << 32) == 32 and T.bits_for((1 << 24) + 1) == 25


@pytest.mark.parametrize("bits", [3, 9, 17, 22, 23, 24, 25, 31, 32])
def test_monotone_map_is_increasing_and_reaches_the_width(bits):
    s = scenes.demo_scene(4, 3) if bits == 3 else _sleepy_scene()
    r, m = T.monotone(s, bits, seed=bits)
    f = m.f.astype(np.float64)
    assert (np.diff(f) > 0).all() and int(m.f[-1]) == (1 << bits) - 1 and int(m.f[0]) < 8
    assert T.tagbits(r) == bits
    t = np.array([3 | (7 << 32), 0 | (2 << 32)], np.uint64)
    assert np.array_equal(m.pair(t), m.f[[3, 0]] | (m.f[[7, 2]] << np.uint64(32)))


def test_permuted_and_shared_premises():
    s = _pile()
    r, m = T.permuted(s, seed=3)
    t = T.collider_tags(r)
    assert len(np.unique(t)) == len(t) and t.max() == 0xffff and t[0] != t.min() and T.tagbits(r) == 16
    c = T.compound(s, np.arange(1, 101, 3))
    sh = T.shared(c)
    body = np.concatenate([sh.box_transforms["body"], sh.sphere_transforms["body"]])
    tag = T.collider_tags(sh)
    for b in np.unique(body):
        assert len(np.unique(tag[body == b])) == 1          # all colliders of a body share one tag
    assert len(np.unique(tag)) < len(np.unique(body))       # and unrelated bodies share tags
    o = _oracle(sh, _cap(sh))
    seen = 0
    for _ in range(20):
        o.step()
        seen = max(seen, T.equal_tag_contacts(o.contact_tags[:o.contacts.count]))
    assert seen > 0, "no touching pair with A == B"


@pytest.mark.parametrize("name", ["permuted_sleeping_islands", "permuted_sleeping_custom_contacts"])
def test_sleeping_cases_reach_the_sleeping_pair_sort_and_the_culled_cache(name):
    seen = []
    case = CASES[name]
    _run(case.scene, case.steps, case.sleep_at, case.high, case.seed, seen)(_oracle, True)
    assert max(s for s, _ in seen) > 0 and max(c for _, c in seen) > 0


def test_custom_contacts_leave_the_collider_range():
    s = _pile()
    o = _oracle(s, _cap(s))
    o.step(); o.collide()
    rows = T.custom_contacts(o, 1, HIGH16, 6)
    assert len(rows) >= 5 and (rows["b"] == 0).any() and (rows["b"] != 0).any()
    assert (rows["A"] > T.collider_tags(s).max()).all() and (rows["A"] > rows["B"]).any() and (rows["A"] < rows["B"]).any()
    n = o.contacts.count
    T.append_wide(o, rows)
    assert o.contacts.count == n + len(rows)
