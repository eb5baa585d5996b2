"""The CUDA narrowphase on the edge-case scenes of tests/np_edge_cases.py: collide() must equal what the unmodified reference recorded
in tests/golden/np_edge_cases.npz bit for bit, and two full steps must equal the CPU oracle at every stage (parity_util), so the
solver sees these contacts too.  Many mixed pairs run per launch: face, edge and no-contact box-box pairs share warps in k_np_clip,
and the tail scenes end on partial warps.  Each tail scene runs a second time with a pair capacity just above its pair count, which
shrinks the narrowphase grids (GRID(max_pairs)) so that k_np_faces, k_np_clip and k_np_emit take several grid-stride rounds.

NaN rule: in the one case that makes NaN contacts on purpose (box-sphere "corner l2 underflows"), the contact data and every solver
stage after it (rows, warm-start states, momentum, states, impulses, cache data, transforms) are compared with any NaN equal to any
NaN; all other bits, and all other scenes, must match exactly."""
import os
import numpy as np
import pytest
import nudge_b200
from tests import np_edge_cases as E
from tests.parity_util import Report, compare_oracle_gpu_step, nan_canonical

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "np_edge_cases.npz")
SCENES = {es.name: es for es in E.all_scenes()}
TAILS = ["tail_%d" % n for n in E.TAILS]


def _cap(es):
    return max(1024, 16 * es.scene.n_colliders)


def _collide_check(es, sim):
    sim.collide()
    sim.download_contacts()
    assert sim.counts().overflow == 0
    view = sim.contacts_view()
    if es.nan_blind:
        view["data"] = nan_canonical(view["data"])
    want = E.golden_of(np.load(GOLDEN), es)
    if es.nan_blind:
        want["data"] = nan_canonical(want["data"])
    errs = E.collide_differences(es, want, view)
    assert not errs, "\n".join(errs)


@pytest.mark.parametrize("name", list(SCENES))
def test_collide_equals_reference(name):
    es = SCENES[name]
    _collide_check(es, nudge_b200.Sim(es.scene, contact_capacity=_cap(es), debug=True))


@pytest.mark.parametrize("name", TAILS)
def test_collide_equals_reference_in_several_grid_stride_rounds(name):
    es = SCENES[name]
    n_pairs = len(es.clusters)   # one broadphase pair per cluster
    sim = nudge_b200.Sim(es.scene, contact_capacity=_cap(es), pair_capacity=n_pairs + 1, debug=True)
    _collide_check(es, sim)
    assert sim.pairs_view()["lo"].shape == (n_pairs,)


@pytest.mark.parametrize("name", list(SCENES))
def test_two_steps_equal_oracle(name):
    from oracle import pyoracle
    es = SCENES[name]
    o = pyoracle.OracleSim(es.scene, contact_capacity=_cap(es))
    g = nudge_b200.Sim(es.scene, contact_capacity=_cap(es), debug=True)
    for i in range(2):
        rep = Report("%s step %d" % (name, i), nan_blind=es.nan_blind)
        assert compare_oracle_gpu_step(o, g, rep), str(rep)
        assert g.counts().overflow == 0
