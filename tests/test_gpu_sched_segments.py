"""The segmented scheduler replay on the GPU (k_sched_spec / k_sched_join / k_sched_merge, k_schedule for buckets that fall back)
against the plain-Python sequential restatement (tests/sched_ref.py) and the CPU oracle."""
import numpy as np
import pytest

import nudge_b200
from nudge_b200 import scenes
from tests import sched_ref

pytestmark = pytest.mark.gpu


def schedule_matches_restatement(g):
    cab = g.debug("cab", np.uint32).reshape(-1, 2)
    batch, lane = sched_ref.schedule_sequential(cab)
    got = g.debug("batch_of", np.uint32).astype(np.int64)
    slot = g.debug("slot_idx", np.uint32).astype(np.int64)
    assert len(got) == len(cab)
    assert (got == batch).all()
    assert (slot == batch * 8 + lane).all()
    return len(cab)


@pytest.mark.parametrize("boxes", [8191, 65536])
def test_large_piles_segment_without_fallback(boxes):
    g = nudge_b200.Sim(scenes.box_drop(boxes, iterations=8, seed=2), debug=True)
    for _ in range(400):
        g.step()
    g.collide(); g.apply_gravity_damping(); g.read_cached_impulses(); g.setup_contact_constraints()
    n = schedule_matches_restatement(g)
    assert n > 16 * 2 * 256   # several segments per bucket
    assert g.debug_scalar("sched_fallback") == 0
    assert g.counts().overflow == 0


def test_hub_platform_falls_back_and_keeps_oracle_parity():
    from oracle import pyoracle
    from tests.parity_util import Report, compare_oracle_gpu_step
    s = scenes.hub_platform(55)
    o = pyoracle.OracleSim(s)
    g = nudge_b200.Sim(s, contact_capacity=o.cap, debug=True)
    fell_back = 0
    for i in range(3):
        rep = Report("hub step %d" % i)
        assert compare_oracle_gpu_step(o, g, rep), str(rep)
        fell_back += g.debug_scalar("sched_fallback")
    assert fell_back > 0


def test_fewer_contacts_than_segments():
    g = nudge_b200.Sim(scenes.demo_scene(2, 2), debug=True)
    for _ in range(40):
        g.step()
    g.collide(); g.apply_gravity_damping(); g.read_cached_impulses(); g.setup_contact_constraints()
    schedule_matches_restatement(g)
