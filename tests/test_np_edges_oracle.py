"""Pins the widened CPU restatement (oracle/nudge_oracle.cpp) on the narrowphase edge cases of tests/np_edge_cases.py: its collide()
output and the stage digests of two full steps must equal what the unmodified reference recorded in tests/golden/np_edge_cases.npz
(tests/golden/make_np_edge_golden.py), bit for bit, NaN bit patterns included.  CPU only."""
import os
import numpy as np
import pytest
from tests import np_edge_cases as E
from tests.parity_util import stage_digests

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "np_edge_cases.npz")
SCENES = {es.name: es for es in E.all_scenes()}


def _oracle(es):
    from oracle import pyoracle
    return pyoracle.OracleSim(es.scene, contact_capacity=max(1024, 16 * es.scene.n_colliders))


@pytest.mark.parametrize("name", list(SCENES))
def test_oracle_collide_and_two_steps_equal_reference(name):
    es = SCENES[name]
    g = np.load(GOLDEN)
    want = E.golden_of(g, es)
    o = _oracle(es)
    o.collide()
    errs = E.collide_differences(es, want, o.contacts_view())
    assert not errs, "\n".join(errs)
    labels, got = stage_digests(_oracle(es), True, 2, nan_blind=es.nan_blind)
    assert list(labels) == list(g["stage_labels"]) and got.shape == want["digests"].shape
    bad = np.nonzero((got != want["digests"]).any(axis=1))[0]
    assert not len(bad), "%s: %d of %d stages differ from the reference, first: %s" % (name, len(bad), len(got), labels[bad[0]])


def test_every_family_and_manifold_size_is_recorded():
    """The fixture keeps the coverage the cases were designed for: every family appears, designed contacts happen, every box-box
    manifold size from 1 to 8 occurs, and the contact data holds subnormal values and NaNs."""
    g = np.load(GOLDEN)
    sizes, n_sub, n_nan, families = set(), 0, 0, set()
    for es in SCENES.values():
        want = E.golden_of(g, es)
        cl = es.cluster_of_tag()[((want["tags"] >> np.uint64(32)) & np.uint64(0xffff)).astype(np.int64)]
        per = np.bincount(cl, minlength=len(es.clusters))
        for j, c in enumerate(es.clusters):
            families.add(c["family"])
            m = int(per[j])
            if c["touch"] is True:
                assert m > 0, "%s made no contact" % es.describe(j)
            elif c["touch"] is False:
                assert m == 0, "%s made %d contacts" % (es.describe(j), m)
            else:
                assert m == c["touch"], "%s made %d contacts, not %d" % (es.describe(j), m, c["touch"])
            if m and all(col["shape"] == "box" for col in c["colliders"]):
                sizes.add(m)
        f = want["data"].view(np.float32)
        n_sub += int(((f != 0) & (np.abs(f) < np.finfo(np.float32).tiny)).sum()); n_nan += int(np.isnan(f).sum())
    assert sizes >= set(range(1, 9)) and n_sub > 0 and n_nan > 0
    assert len(families) >= 30
