"""CPU checks of oracle/jacobi_ref.py (the restatement the throughput-mode solver is tested against) against the C oracle, which is
pinned bit-for-bit to the compiled reference: (1) with every body counted once the mass split must reproduce the reference's
effective-mass planes (nudge.cpp:4350-4561), (2) on a scene where no body has two contacts a Jacobi pass IS a Gauss-Seidel sweep,
so it must reproduce apply_impulses (nudge.cpp:4640-4855) up to the reference's rcpps/rsqrtps approximation error."""
import numpy as np
from nudge_b200 import scenes
from oracle import pyoracle, jacobi_ref as J


def _rows41(o):
    v = o.constraints_view()
    c = v["contact"]
    n = o.contacts.count
    first = np.full(n, -1, np.int64)
    for lane in range(len(c) - 1, -1, -1):      # first lane of every contact (leftover batches repeat lane 0)
        if c[lane] < n: first[c[lane]] = lane
    assert (first >= 0).all()
    a, b = v["a"][first].astype(np.int64), v["b"][first].astype(np.int64)
    P = np.zeros((41, n), np.float32)
    P[:39] = v["rows"][first].T
    P[39] = o.properties["mass_inverse"][a]; P[40] = o.properties["mass_inverse"][b]
    return P, v["states"][first].T.copy(), a, b


def _setup(o):
    o.collide(); o.apply_gravity_damping(); o.read_cached_impulses(); o.setup_contact_constraints()


def test_split_with_unit_counts_reproduces_the_reference_planes():
    o = pyoracle.OracleSim(scenes.demo_scene(120, 120, iterations=4, spread=3.0, height=12.0))
    for _ in range(60):
        o.step()
    _setup(o)
    P, st, a, b = _rows41(o)
    assert P.shape[1] > 200
    t = J.split_terms(P, a, b, np.ones(o.scene.n_bodies, np.int64))
    for k in ("NVTNI", "BIAS", "FC_X", "FC_Y", "FC_Z"):
        want = P[J.IX[k]].astype(np.float64)
        scale = np.abs(want).max()
        assert np.abs(t[k] - want).max() <= 2e-5 * scale, k


def test_jacobi_pass_absolute_sums_add_every_contact_change_once():
    """abs_sums (the per-body rounding scale of the kernel's free-order float32 sums): equal to the per-contact velocity changes, read
    off a pass in which every contact side gets a private copy of its body, taken absolute and added per real body."""
    o = pyoracle.OracleSim(scenes.demo_scene(120, 120, iterations=4, spread=3.0, height=12.0))
    for _ in range(60):
        o.step()
    _setup(o)
    P, st, a, b = _rows41(o)
    n, B = P.shape[1], o.scene.n_bodies
    lin, ang = o.momentum["velocity"].astype(np.float64), o.momentum["angular_velocity"].astype(np.float64)
    for warm in (True, False):
        imp = o.impulses_view()["data"]["impulse"] if warm else None
        l1, w1, s1, alin, aang = J.jacobi_pass(P, st, a, b, lin, ang, warm=warm, impulses=imp, abs_sums=True)
        l0, w0, s0 = J.jacobi_pass(P, st, a, b, lin, ang, warm=warm, impulses=imp)
        assert np.array_equal(l0, l1) and np.array_equal(w0, w1) and np.array_equal(s0, s1)
        # private copies: side a of contact k is body 1 + 2k, side b is 2 + 2k (the world stays body 0)
        pa, pb = np.where(a != 0, 1 + 2 * np.arange(n), 0), np.where(b != 0, 2 + 2 * np.arange(n), 0)
        plin, pang = np.zeros((1 + 2 * n, 3)), np.zeros((1 + 2 * n, 3))
        plin[pa], pang[pa], plin[pb], pang[pb] = lin[a], ang[a], lin[b], ang[b]
        ql, qw, _ = J.jacobi_pass(P, st, pa, pb, plin, pang, warm=warm, impulses=imp)
        want_l, want_w = np.zeros((B, 3)), np.zeros((B, 3))
        np.add.at(want_l, np.concatenate([a, b]), np.abs(ql - plin)[np.concatenate([pa, pb])])
        np.add.at(want_w, np.concatenate([a, b]), np.abs(qw - pang)[np.concatenate([pa, pb])])
        want_l[0] = 0; want_w[0] = 0
        eps = 1e-12 * max(1.0, np.abs(lin).max(), np.abs(ang).max())    # (v + d) - v is d up to float64 rounding of v
        assert np.abs(alin - want_l).max() <= eps and np.abs(aang - want_w).max() <= eps
        assert (np.abs(l1 - lin) <= alin + eps).all() and (np.abs(w1 - ang) <= aang + eps).all()
        assert alin.max() > 1e-3 and (np.bincount(np.concatenate([a, b]), minlength=B)[1:] > 1).any()


def test_jacobi_pass_equals_a_gauss_seidel_sweep_when_no_body_has_two_contacts():
    n = 36
    s = scenes.demo_scene(0, n, iterations=1)
    k = np.arange(n)
    s.transforms["position"][1:, 0] = (k % 6) * 4.0; s.transforms["position"][1:, 2] = (k // 6) * 4.0
    s.transforms["position"][1:, 1] = -10.0 + s.sphere_data["radius"] - 0.02      # resting on the ground box (top at y = -10), slightly sunk
    rng = np.random.default_rng(4)
    s.momentum["velocity"][1:] = rng.normal(size=(n, 3)) * 0.3; s.momentum["angular_velocity"][1:] = rng.normal(size=(n, 3)) * 0.3
    o = pyoracle.OracleSim(s)
    _setup(o)
    P, st, a, b = _rows41(o)
    assert P.shape[1] == n and len(np.unique(np.concatenate([a[a != 0], b[b != 0]]))) == n
    lin0, ang0 = o.momentum["velocity"].copy(), o.momentum["angular_velocity"].copy()
    o.apply_impulses()
    lin1, ang1, st1 = J.jacobi_pass(P, st, a, b, lin0, ang0)
    assert np.abs(lin1 - o.momentum["velocity"]).max() < 2e-3 and np.abs(ang1 - o.momentum["angular_velocity"]).max() < 2e-3
    assert np.abs(lin1 - lin0).max() > 1e-2       # the sweep did something
    _, st_ref, _, _ = _rows41(o)
    assert np.abs(st1 - st_ref).max() < 2e-3 * max(1.0, np.abs(st_ref).max())
