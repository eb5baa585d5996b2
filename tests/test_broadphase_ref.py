"""Pins the CPU oracle's broadphase on the edge-case geometry of tests/broadphase_edges.py before the GPU is held to it: on every scene the
oracle's pair set (an independent sort-and-sweep) equals every strictly overlapping AABB pair (tests/grid_ref.brute_pairs), the grid
restatement's premises hold (far scenes sit at the intended distance, the tight pair straddles a cell boundary with a quantised span of at
most 2^j - 1, boundary spheres need the designed level and land on the designed side of the grid level, each connection of the
feature scenes joins the bodies of an overlapping pair that only the connected opt-out removes, wrapped corners quantise past 65535), and on every scene without filters, sensors or
kinematic bodies two full steps of the oracle equal the unmodified reference's stage digests in tests/golden/broadphase_edges.npz
(tests/golden/make_broadphase_golden.py).  CPU only."""
import os
import numpy as np
import pytest
from tests import broadphase_edges as E, grid_ref as G
from tests.parity_util import stage_digests

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "broadphase_edges.npz")


@pytest.fixture(scope="module")
def edge_scenes():
    return {es.name: es for es in E.all_scenes(G.host_rcp())}


NAMES = ["far_2^%d" % e for e in E.FAR_EXPONENTS] + ["boundary_%s_%d" % (s, n) for s in ("at", "below", "above") for n in (63, 64)] + \
    ["large_%d_dynamic" % n for n in E.LARGE_COUNTS] + ["large_%d_%s" % (n, v) for n in (64, 200) for v in ("features", "kinematic")] + \
    ["one_cell_level16", "one_cell_beyond", "flat_layer", "same_corner_12", "alone_1", "alone_2", "wrapped", "multi_scale"]


def check_premise(es, g):
    """Asserts what the scene was built to exercise, from the grid restatement g (grid_ref.Grid of its colliders)."""
    p = es.premise
    small_span = g.span()[g.small]
    assert (small_span <= (1 << g.j) - 1).all(), "%s: a small collider spans more than its cell" % es.name
    if "scaled_min" in p:
        lo, hi = p["scaled_min"]
        assert lo <= g.max_scaled_min() < hi
        a, b = p["tight_pair"]
        assert g.small[a] and g.small[b] and g.j == p["level"]
        assert g.span()[a, 0] >= (1 << g.j) - 64, "the constructed collider does not fill its cell"   # float positions 2^28 units out step by ~17 units
        # b's min corner lies one float inside a's far face, in the next cell: the pair overlaps strictly
        assert g.cell()[b, 0] == g.cell()[a, 0] + 1 and np.nextafter(g.lo[b, 0], np.float32(np.inf)) >= g.hi[a, 0]
        assert (g.hi[b] > g.lo[a]).all() and (g.hi[a] > g.lo[b]).all()
    if "boundary" in p:
        first, level, j, small = p["boundary"]
        assert (g.levels[first:] == level).all() and g.j == j and (g.small[first:] == small).all()
        if not es.name.startswith("boundary_above"):   # at the bound (or one ulp under it): a sphere fills its cell
            assert g.span()[first:].max() >= (1 << j) - 8
    if "large_count" in p:
        n = p["large_count"]
        if n <= 64:
            assert g.n_large == n
        else:
            assert g.small[p["slabs"]].all() and g.n_large < 64
    if es.name.startswith("one_cell"):
        assert g.j == 16 and (g.n_large > 64) == es.name.endswith("beyond")
    if "connected" in p:   # each connection removes an overlapping pair that passes the filter and holds no sensor
        body = np.concatenate([es.scene.box_transforms["body"], es.scene.sphere_transforms["body"]]).astype(np.int64)
        f, sens, pairs = es.scene.collision_filters, es.scene.sensors, G.brute_pairs(g.lo, g.hi)
        slabs = set(p["slabs"].tolist())
        for (a, b), c in zip(p["connected"], es.scene.connections):
            assert (a, b) in pairs and {body[a], body[b]} == {int(c["a"]), int(c["b"])}
            assert f["category"][a] & f["mask"][b] and f["category"][b] & f["mask"][a] and not sens[a] and not sens[b]
        (a0, b0), (a1, b1) = p["connected"]
        assert (a0 in slabs) != (b0 in slabs) and a1 in slabs and b1 in slabs
        assert es.scene.filter_flags & 1
    if "flat_axis" in p:
        assert g.frame.smin[p["flat_axis"]] == g.frame.smax[p["flat_axis"]]
    if p.get("all_large") or es.name.startswith("alone"):
        assert g.n_large == es.scene.n_colliders
    if "wrapped" in p:
        w = p["wrapped"]
        assert (g.q_lo[w, 0] >= 65536).all() and not g.small[w].any()


def oracle_for(es):
    from oracle import pyoracle
    from tests.kinematic_ref import KinematicOracleSim
    from tests.sensor_ref import SensorOracleSim
    cls = {"features": SensorOracleSim, "kinematic": KinematicOracleSim}.get(es.kind, pyoracle.OracleSim)
    return cls(es.scene, contact_capacity=E.CAPACITY)


def test_every_family_is_covered(edge_scenes):
    assert sorted(edge_scenes) == sorted(NAMES)


@pytest.mark.parametrize("name", NAMES)
def test_oracle_pairs_equal_brute_force_and_premises_hold(name, edge_scenes):
    from oracle import pyoracle
    es = edge_scenes[name]
    g = G.Grid.of_scene(es.scene, G.host_rcp())
    check_premise(es, g)
    o = pyoracle.OracleSim(es.scene, contact_capacity=E.CAPACITY)   # the plain oracle: every overlapping pair, before any filter
    o.collide()
    v = o.pairs_view()
    assert G.pair_set(v["lo"], v["hi"]) == G.brute_pairs(g.lo, g.hi)
    assert len(v["lo"]) == len(G.pair_set(v["lo"], v["hi"]))   # each pair once


@pytest.mark.parametrize("name", [n for n in NAMES if not n.endswith(("features", "kinematic"))])
def test_oracle_two_steps_equal_reference(name, edge_scenes):
    es = edge_scenes[name]
    gold = np.load(GOLDEN)
    assert es.scene.fits_reference()
    assert np.array_equal(E.input_digest(es.scene), gold[name + "/inputs"]), "the scene is not the one the reference ran"
    labels, got = stage_digests(oracle_for(es), True, 2)
    want = gold[name + "/digests"]
    assert list(labels) == list(gold["stage_labels"]) and got.shape == want.shape
    bad = np.nonzero((got != want).any(axis=1))[0]
    assert not len(bad), "%s: %d of %d stages differ from the reference, first: %s" % (name, len(bad), len(got), labels[bad[0]])


def test_tight_span_bound_holds_ulp_by_ulp_far_from_the_origin():
    """The quantisation is one rounding of a value below 65536, so the quantised span of a collider that passes the float test at level j
    never exceeds 2^j - 1, at any distance: boxes of every size near the boundary of levels 4 to 14, stepped ulp by ulp in position, on
    frames whose min corner lies 2^16 to 2^28 quantised units from the origin."""
    rcp = G.host_rcp()
    rng = np.random.default_rng(3)
    for e in (16, 20, 24, 26, 28):
        d = np.float32(2.0 ** e / 2184.0)
        anchor_lo = np.array([[d, d, d], [d + 30.0, d + 30.0, d + 30.0]], np.float32)
        fr = G.Frame(anchor_lo, rcp)
        L = float(fr.L[0])
        for l in range(4, 15):
            h = np.float32(((1 << l) - 2) / L / 2.0)
            c = np.repeat((d + rng.uniform(1.0, 29.0, (64, 1)) + np.zeros((1, 3))).astype(np.float32), 96, axis=0)
            x = np.ascontiguousarray(c[:, 0])
            c[:, 0] = (x.view(np.int32) + np.tile(np.arange(96, dtype=np.int32), 64)).view(np.float32)   # 96 consecutive floats each
            hh = (h * (1.0 + rng.uniform(-1.0, 1.0, len(c)) * min(0.5, max(1e-3, 64.0 / (1 << l))))).astype(np.float32)
            lo, hi = c - hh[:, None], c + hh[:, None]
            ok = G.level_needed(lo, hi, L) <= l
            assert ok.any() and (~ok).any()
            span = fr.quantise(hi[ok]).astype(np.int64) - fr.quantise(lo[ok]).astype(np.int64)
            assert span.max() <= (1 << l) - 1, (e, l, span.max())
