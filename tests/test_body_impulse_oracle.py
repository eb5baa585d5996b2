"""The body-impulse restatement (tests/impulse_ref.py) on the CPU: it agrees with the float64 rigid-body formulas, duplicates applied in order
differ from their float sum only in rounding, and on the oracle a hit on one body of a sleeping pile wakes exactly that pile's island at the
next collide.  CPU only."""
import numpy as np
from nudge_b200 import scenes
from tests.impulse_ref import apply_body_impulses, apply_radial_impulse, world_inverse_inertia, random_impulses


def _bodies(n, seed):
    rng = np.random.default_rng(seed)
    s = scenes.demo_scene(n // 2, n - n // 2, seed=seed)
    s.transforms["rotation"][1:] = scenes._random_unit_quaternions(rng, s.n_bodies - 1)
    s.momentum["velocity"] = rng.normal(0.0, 1.0, (s.n_bodies, 3))
    s.momentum["angular_velocity"] = rng.normal(0.0, 1.0, (s.n_bodies, 3))
    s.idle[:] = rng.integers(0, 256, s.n_bodies)
    from nudge_b200 import abi
    return abi.HostState(s), rng


def _quat_matrix64(q):
    x, y, z, w = q
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                     [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                     [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])


def _close(got, want, rel=1e-5):
    scale = max(np.abs(want).max(), 1e-30)
    assert np.abs(np.asarray(got, np.float64) - want).max() <= rel * scale, (got, want)


def test_restatement_agrees_with_float64_rigid_body_formulas():
    st, rng = _bodies(200, 7)
    for b in range(1, st.scene.n_bodies):
        R = _quat_matrix64(st.transforms["rotation"][b].astype(np.float64))
        Iw = R @ np.diag(st.properties["inertia_inverse"][b].astype(np.float64)) @ R.T
        W = world_inverse_inertia(st.transforms["rotation"][b:b + 1], st.properties[b:b + 1])[0].astype(np.float64)
        _close(W, np.array([Iw[0, 0], Iw[1, 1], Iw[2, 2], Iw[0, 1], Iw[0, 2], Iw[1, 2]]))
    rows = random_impulses(rng, np.arange(1, st.scene.n_bodies), 150, duplicates=False, zeros=0.0)
    v0, w0 = st.momentum["velocity"].astype(np.float64), st.momentum["angular_velocity"].astype(np.float64)
    apply_body_impulses(st, rows)
    for r in rows:
        b = int(r["body"])
        R = _quat_matrix64(st.transforms["rotation"][b].astype(np.float64))
        Iw = R @ np.diag(st.properties["inertia_inverse"][b].astype(np.float64)) @ R.T
        J, o, L = (r[f].astype(np.float64) for f in ("impulse", "offset", "angular_impulse"))
        _close(st.momentum["velocity"][b] - v0[b], float(st.properties["mass_inverse"][b]) * J)
        _close(st.momentum["angular_velocity"][b] - w0[b], Iw @ (np.cross(o, J) + L), rel=2e-5)   # the difference of two float32 sums
    assert (st.idle[rows["body"]] == 0).all()


def test_explosion_follows_the_linear_falloff_law():
    st, rng = _bodies(400, 8)
    center, radius, impulse = np.float32([0.5, 100.0, -0.25]), np.float32(120.0), np.float32(7.5)
    v0 = st.momentum["velocity"].astype(np.float64)
    idle0 = st.idle.copy()
    hit = apply_radial_impulse(st, center, radius, impulse)
    d = st.transforms["position"].astype(np.float64) - center.astype(np.float64)
    dist = np.linalg.norm(d, axis=1)
    assert hit.sum() > 50 and (~hit[1:]).sum() > 50 and not hit[0]
    assert np.array_equal(hit[1:], dist[1:] < 120.0)
    for b in np.nonzero(hit)[0]:
        J = float(impulse) * (1.0 - dist[b] / float(radius)) * d[b] / dist[b]
        _close(st.momentum["velocity"][b] - v0[b], float(st.properties["mass_inverse"][b]) * J, rel=2e-5)
    assert (st.idle[hit] == 0).all() and np.array_equal(st.idle[~hit], idle0[~hit])
    assert np.array_equal(st.momentum["velocity"][~hit], v0[~hit].astype(np.float32))


def test_duplicates_in_order_differ_from_their_sum_only_in_rounding():
    a, rng = _bodies(50, 9)
    b, _ = _bodies(50, 9)
    rows = random_impulses(rng, [5], 6, zeros=0.0)
    apply_body_impulses(a, rows)
    summed = rows[:1].copy()
    summed["offset"] = 0
    summed["impulse"] = rows["impulse"].sum(0, dtype=np.float32)
    summed["angular_impulse"] = (np.cross(rows["offset"].astype(np.float32), rows["impulse"]) + rows["angular_impulse"]).sum(0, dtype=np.float32)
    apply_body_impulses(b, summed)
    for f in ("velocity", "angular_velocity"):
        x, y = a.momentum[f][5].astype(np.float64), b.momentum[f][5].astype(np.float64)
        assert np.abs(x - y).max() <= 1e-5 * max(np.abs(y).max(), 1.0)
    others = np.arange(50 + 1) != 5
    assert np.array_equal(a.momentum[others], b.momentum[others])


def two_piles(height=6):
    """Two columns of boxes (with a sphere on top) resting on the ground, 30 apart: two islands.  Returns the scene and each pile's bodies."""
    n = height
    pos = []
    for x0 in (-15.0, 15.0):
        for k in range(n):
            pos.append((x0 + 0.02 * (k % 2), 0.5 + 0.99 * k, 0.0))
    pos = np.array(pos, np.float32)
    sizes = np.full((2 * n, 3), 0.5, np.float32)
    sph = np.array([(-15.0, 0.5 + 0.99 * n + 0.45, 0.0), (15.0, 0.5 + 0.99 * n + 0.45, 0.0)], np.float32)
    s = scenes._assemble("two_piles", sizes, pos, None, np.float32([0.5, 0.5]), sph, ground_half=(400.0, 10.0, 400.0), ground_y=-10.0)
    s.iterations = 8
    a = [1 + k for k in range(n)] + [1 + 2 * n]
    b = [1 + n + k for k in range(n)] + [2 + 2 * n]
    return s, np.array(a), np.array(b)


def settle_and_sleep(sim, steps=120):
    """Steps `sim` (an OracleSim or a Sim through its stage calls) and puts every body to sleep at rest."""
    for _ in range(steps):
        sim.collide(); sim.apply_gravity_damping(); sim.read_cached_impulses(); sim.setup_contact_constraints()
        for _ in range(int(sim.scene.iterations)):
            sim.apply_impulses()
        sim.update_cached_impulses(); sim.write_cached_impulses(); sim.advance()
    if hasattr(sim, "download_bodies"):
        sim.download_bodies()
    sim.idle[1:] = 0xff
    sim.momentum["velocity"][1:] = 0; sim.momentum["angular_velocity"][1:] = 0
    if hasattr(sim, "upload_bodies"):
        sim.upload_bodies()


def test_a_hit_wakes_exactly_its_island_at_the_next_collide_on_the_oracle():
    from oracle import pyoracle
    s, pile_a, pile_b = two_piles()
    o = pyoracle.OracleSim(s)
    settle_and_sleep(o)
    o.collide()
    assert len(o.contacts_view()["active"]) == 0 and len(o.contacts_view()["sleeping"]) > 0
    before_b = (o.transforms[pile_b].copy(), o.momentum[pile_b].copy(), o.idle[pile_b].copy())
    hit = np.zeros(1, scenes.BODY_IMPULSE)
    hit["body"] = pile_a[2]; hit["impulse"] = (0.5, 0.0, 0.0); hit["offset"] = (0.0, 0.3, 0.0)
    apply_body_impulses(o, hit)
    assert o.idle[pile_a[2]] == 0 and (o.idle[pile_b] == 0xff).all()
    o.collide()
    assert np.array_equal(np.sort(o.contacts_view()["active"]), np.sort(pile_a))
    assert np.array_equal(o.transforms[pile_b], before_b[0]) and np.array_equal(o.momentum[pile_b], before_b[1]) and np.array_equal(o.idle[pile_b], before_b[2])
