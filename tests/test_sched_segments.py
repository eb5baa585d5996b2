"""The segmented scheduler replay (speculative runs, joins, fall-back; tests/sched_ref.py and nb_solver.cuh above k_schedule) gives
the same batch and lane for every contact, hence the same emission order, as the sequential replay."""
import numpy as np
import pytest

from tests import sched_ref


def pile_like(n, seed, conflicts):
    """Body pairs like a settled pile's: mostly distinct bodies within reach of one slot, with `conflicts` contacts that share a
    body with a contact 1-3 bucket positions earlier."""
    rng = np.random.default_rng(seed)
    cab = np.stack([np.arange(n) * 2 + 1, np.arange(n) * 2 + 2], 1)
    if conflicts:
        idx = rng.integers(64, n, size=conflicts)
        cab[idx, 0] = cab[idx - 16 * rng.integers(1, 4, size=conflicts), rng.integers(0, 2, size=conflicts)]
    return cab


def check(cab, segs, seg_len, cap=64, expect_fallback=None):
    ref_b, ref_l = sched_ref.schedule_sequential(cab)
    b, l, fb = sched_ref.schedule_segmented(cab, segs, seg_len, cap=cap)
    assert (b == ref_b).all() and (l == ref_l).all()
    if expect_fallback is not None:
        assert (fb > 0) == expect_fallback
    return fb


@pytest.mark.parametrize("seed", range(4))
@pytest.mark.parametrize("segs", [2, 8, 32])
def test_pile_like_sequences_couple_and_match(seed, segs):
    n = 16 * 1500
    check(pile_like(n, seed, n // 20), segs, (n // 16 + segs - 1) // segs, expect_fallback=False if segs <= 8 else None)


@pytest.mark.parametrize("seed", range(3))
def test_random_sequences_match(seed):
    rng = np.random.default_rng(seed)
    for nb in (30, 400, 5000):
        cab = rng.integers(1, nb, size=(3000, 2))
        check(cab, 4, (3000 // 16 + 3) // 4)


def test_hub_sequences_fall_back_and_match():
    # one body in every contact: each contact opens its own slot, the list outgrows the cap
    n = 16 * 300
    cab = np.stack([np.full(n, 7), np.arange(n) + 10], 1)
    assert check(cab, 4, 75, cap=64, expect_fallback=True) == 16


@pytest.mark.parametrize("n", [0, 1, 7, 15, 16, 17, 100])
def test_tiny_scenes(n):
    cab = pile_like(max(n, 1), 1, 0)[:n].reshape(-1, 2)
    check(cab, 1, (n + 15) // 16)
    if n:
        check(cab, 2, max(1, (n + 15) // 32))


def test_segment_shorter_than_a_slot():
    n = 16 * 20
    check(pile_like(n, 2, 10), 8, 3)


def test_couple_at_the_segment_start_and_after_the_first_empty_list():
    n = 16 * 64
    cab = pile_like(n, 3, 0)
    # segment start at 32 with a conflict-free stream: the previous segment ends with an empty list (no join), and a segment
    # start at 36 carries a half slot: the join couples with run 4 after the first 4 contacts, where its list first empties
    check(cab, 2, 32, expect_fallback=False)
    check(cab, 2, 36, expect_fallback=False)
    stats = {}
    sched_ref.schedule_segmented(cab, 2, 36, cap=64, stats=stats)
    assert max(stats["join_len"]) == 4


def test_join_couples_at_the_last_contact_of_its_segment():
    # 36 conflict-free contacts leave segment 0 with a half slot; segment 1 holds the last 4 contacts of the bucket, which fill it:
    # the join's list empties only after the segment's last contact, where it couples with run 4 (which starts there, empty)
    cab = pile_like(16 * 40, 3, 0)
    stats = {}
    b, l, fb = sched_ref.schedule_segmented(cab, 2, 36, cap=64, stats=stats)
    ref_b, ref_l = sched_ref.schedule_sequential(cab)
    assert fb == 0 and (b == ref_b).all() and (l == ref_l).all()
    assert stats["join_len"] == [4] * 16   # = the length of segment 1


def test_one_phase_per_segment_cannot_couple_after_a_partial_slot():
    # the same pile with only run 0 per segment: the carried half slot keeps the join 4 contacts out of phase with run 0
    cab = pile_like(16 * 200, 4, 0)
    b, l, fb = sched_ref.schedule_segmented(cab, 2, 100, cap=64, phases=1)
    assert fb == 16
    b8, l8, fb8 = sched_ref.schedule_segmented(cab, 2, 100, cap=64)
    assert fb8 == 0 and (b8 == b).all() and (l8 == l).all()


def test_sequential_restatement_matches_oracle_batches():
    """The sequential restatement against the CPU oracle's schedule on a settling demo pile (the oracle is built by build())."""
    from nudge_b200 import scenes
    from oracle import pyoracle
    from tests.parity_util import rows_by_contact
    o = pyoracle.OracleSim(scenes.demo_scene(600, 600))
    for _ in range(30):
        o.step()
    o.collide(); o.apply_gravity_damping(); o.read_cached_impulses(); o.setup_contact_constraints()
    oc, oi = o.contacts_view(), o.impulses_view()
    n = oc["count"]
    assert n > 16 * 40
    order = oi["sorted"].astype(np.int64)
    bodies = np.stack([oc["bodies"]["a"], oc["bodies"]["b"]], 1)[order]
    cab = sched_ref.body_pairs(bodies)
    batch, _ = sched_ref.schedule_sequential(cab)
    assert (batch == rows_by_contact(o.constraints_view(), n)["batch"][order]).all()
    nbmax = (n + 15) // 16
    for segs in (2, 4):
        b, _, fb = sched_ref.schedule_segmented(cab, segs, (nbmax + segs - 1) // segs, cap=64)
        assert (b == batch).all()
