"""The grid broadphase where its cell-fit rule is tight (tests/broadphase_edges.py; DESIGN.md section 2.3): scenes far from the origin with
the tightest pair the rule allows, extents at a level boundary, 63 to 200 large colliders (dynamic slabs, filters, a sensor zone, a
connected pair, kinematic platforms), a single-cell grid, degenerate frames, wrapped corners and multi-scale colliders.

On every scene: the grid level and large count the device reports (nb_debug_read "grid_level" / "grid_large") are the ones the numpy
restatement (tests/grid_ref.py, with the device's rcpps) derives, so the test exercised the path it was built for; the pair list equals the
CPU oracle's bit for bit and, as a set, every strictly overlapping AABB pair; two full steps equal the oracle stage by stage (filters and
sensors through tests/sensor_ref.py, with the sensor overlaps; several kinematic bodies through tests/kinematic_ref.py, collide stage from
the device's state); graph-replayed nb_steps equal the stage calls; and on the far, large and single-cell scenes seeded rays equal the brute
force of oracle/raycast_ref.py byte for byte."""
import numpy as np
import pytest
import nudge_b200
from nudge_b200 import scenes
from tests import broadphase_edges as E, grid_ref as G
from tests.gpu_util import side_stream
from tests.parity_util import Report, compare_oracle_gpu_step, sync_oracle_from_gpu
from tests.test_broadphase_ref import NAMES, check_premise

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def rcp():
    return nudge_b200.Sim(scenes.two_boxes()).device_rcp


@pytest.fixture(scope="module")
def edge_scenes(rcp):
    return {es.name: es for es in E.all_scenes(rcp)}


def _sim(es, **kw):
    return nudge_b200.Sim(es.scene, contact_capacity=E.CAPACITY, pair_capacity=1 << 16, **kw)


def _grid_before_collide(g, rcp):
    """The restatement of the grid the next collide of g builds (from the transforms g holds on the device)."""
    g.download_bodies()
    return G.Grid(*G.aabbs(g.transforms, g.box_transforms, g.box_data, g.sphere_transforms, g.sphere_data), rcp)


def _check_grid(es, g, gr):
    """The device's grid level and large count of the last collide are the restatement's."""
    assert (g.debug_scalar("grid_level"), g.debug_scalar("grid_large")) == (gr.j, gr.n_large), es.name


@pytest.mark.parametrize("name", NAMES)
def test_pairs_and_two_steps_equal_the_oracle(name, edge_scenes, rcp):
    from oracle import pyoracle
    from tests.kinematic_ref import KinematicOracleSim
    from tests.sensor_ref import SensorOracleSim
    es = edge_scenes[name]
    check_premise(es, G.Grid.of_scene(es.scene, rcp))
    g = _sim(es, debug=True)
    if es.kind == "kinematic":   # several kinematic bodies: the restatement covers the collide stage, from the device's state
        o = KinematicOracleSim(es.scene, contact_capacity=E.CAPACITY)
        for i in range(2):
            gr = _grid_before_collide(g, rcp)
            sync_oracle_from_gpu(o, g)
            o.collide(); g.collide(); g.download_contacts()
            _check_grid(es, g, gr)
            rep = Report("%s step %d" % (name, i))
            op, gp = o.pairs_view(), g.pairs_view()
            rep.eq("pairs.lo", op["lo"], gp["lo"]); rep.eq("pairs.hi", op["hi"], gp["hi"])
            oc, gc = o.contacts_view(), g.contacts_view()
            for fld in ("data", "bodies", "tags", "features", "sleeping", "active"):
                rep.eq(fld, oc[fld], gc[fld])
            assert rep.ok, str(rep)
            assert G.pair_set(gp["lo"], gp["hi"]) <= G.brute_pairs(gr.lo, gr.hi)
            g.apply_gravity_damping(); g.read_cached_impulses(); g.setup_contact_constraints(); g.apply_impulses(int(es.scene.iterations))
            g.update_cached_impulses(); g.write_cached_impulses(); g.advance()
        assert g.counts().overflow == 0
        return
    o = SensorOracleSim(es.scene, contact_capacity=E.CAPACITY) if es.kind == "features" else pyoracle.OracleSim(es.scene, contact_capacity=E.CAPACITY)
    for i in range(2):
        rep = Report("%s step %d" % (name, i))
        gr = _grid_before_collide(g, rcp)
        assert compare_oracle_gpu_step(o, g, rep), str(rep)
        assert g.counts().overflow == 0
        _check_grid(es, g, gr)
        if i == 0:
            gp = g.pairs_view()
            found = G.pair_set(gp["lo"], gp["hi"])
            assert len(found) == len(gp["lo"])
            if es.kind == "features":
                assert found <= G.brute_pairs(gr.lo, gr.hi)
            else:
                assert found == G.brute_pairs(gr.lo, gr.hi)
            if "tight_pair" in es.premise:
                assert tuple(es.premise["tight_pair"]) in found
            for pair in es.premise.get("connected", ()):   # overlapping, passing the filter, and rejected only as connected
                assert pair in G.brute_pairs(gr.lo, gr.hi) and pair not in found
        if es.kind == "features":
            ov = g.sensor_overlaps()
            assert ov.tobytes() == o.overlaps.tobytes(), "%s step %d: %d vs %d overlaps" % (name, i, len(ov), len(o.overlaps))


@pytest.mark.parametrize("name", ["far_2^16", "far_2^28", "boundary_above_63", "large_64_features", "large_200_kinematic", "one_cell_level16",
                                  "one_cell_beyond", "same_corner_12", "wrapped", "multi_scale"])
def test_graph_replayed_steps_equal_the_stage_calls(name, edge_scenes):
    es = edge_scenes[name]
    a, b = _sim(es, stream=side_stream()), _sim(es)
    for i in range(3):
        a.step(); b.step_staged()
        for x in (a, b):
            x.download_bodies()
        assert a.transforms.tobytes() == b.transforms.tobytes() and a.momentum.tobytes() == b.momentum.tobytes() and a.idle.tobytes() == b.idle.tobytes(), i
        assert (a.debug_scalar("grid_level"), a.debug_scalar("grid_large")) == (b.debug_scalar("grid_level"), b.debug_scalar("grid_large"))
    assert a.debug_scalar("graph_records") == 1 and a.counts().overflow == 0


@pytest.mark.parametrize("name", ["far_2^%d" % e for e in E.FAR_EXPONENTS] + ["large_64_dynamic", "large_200_dynamic", "one_cell_level16", "one_cell_beyond"])
def test_rays_equal_the_brute_force(name, edge_scenes):
    from tests.test_gpu_raycast import families, _same
    es = edge_scenes[name]
    sim = _sim(es, stream=side_stream())
    sim.step()
    rng = np.random.default_rng(sum(map(ord, name)))
    hits = 0
    for fam, rays in families(sim, rng, 128).items():
        got = _same(sim, rays, min_hits=0)
        hits += int((got["collider"] != 0xffffffff).sum())
    assert hits > 0
