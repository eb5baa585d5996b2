"""The force-stage restatement (tests/body_force_ref.py) on the CPU: default entries give the bits of the stage without a table, the
restatement agrees with the float64 formulas (free fall with a gravity scale and damping, I^-1 T on rotated boxes, a body-frame force that
turns with the body), and on the oracle a pile at gravity scale 0.5 still sleeps while a body pressed into the ground keeps its island awake
until its force is cleared.  CPU only."""
import numpy as np
from nudge_b200 import abi, scenes
from tests.body_force_ref import BodyForceOracleSim, apply_stage, default_table, qrot, remove_table, add_table
from tests.test_body_impulse_oracle import _quat_matrix64, _close, two_piles

F = np.float32


def _state(n, seed):
    rng = np.random.default_rng(seed)
    s = scenes.demo_scene(n // 2, n - n // 2, seed=seed)
    s.transforms["rotation"][1:] = scenes._random_unit_quaternions(rng, s.n_bodies - 1)
    s.momentum["velocity"] = rng.normal(0.0, 1.0, (s.n_bodies, 3))
    s.momentum["angular_velocity"] = rng.normal(0.0, 1.0, (s.n_bodies, 3))
    s.idle[:] = rng.integers(0, 256, s.n_bodies)
    return abi.HostState(s), rng


def test_default_entries_give_the_bits_of_the_stage_without_a_table():
    for seed, damping in ((1, F(0.25)), (2, F(0.0)), (3, F(-0.0)), (4, F(1.5))):
        a, rng = _state(300, seed)
        for f in ("velocity", "angular_velocity"):   # signed zeros in some components
            z = rng.random((a.scene.n_bodies, 3)) < 0.2
            a.momentum[f][z] = np.where(rng.random(z.sum()) < 0.5, F(0.0), F(-0.0))
        b = abi.HostState(a.scene)
        b.momentum[:] = a.momentum; b.idle[:] = a.idle
        active = np.sort(rng.choice(np.arange(1, a.scene.n_bodies), 200, replace=False)).astype(np.uint32)
        for st in (a, b):
            st.active_indices[:len(active)] = active; st.active.count = len(active)
            st.scene.damping = damping
        a.apply_gravity_damping()
        table = default_table(a.scene.n_bodies)
        table["force"][::3] = -0.0; table["torque"][::5] = (0.0, -0.0, 0.0)   # zero forces are skipped
        table["flags"][::2] = scenes.BODY_FORCE_LOCAL
        pushed = apply_stage(b, table, active, b.scene.time_step, b.scene.gravity, damping)
        assert len(pushed) == 0
        assert a.momentum.tobytes() == b.momentum.tobytes() and a.idle.tobytes() == b.idle.tobytes()


def test_free_fall_with_gravity_scale_and_damping_follows_the_float64_law():
    st, rng = _state(120, 5)
    B = st.scene.n_bodies
    table = default_table(B)
    table["gravity_scale"] = rng.choice([-0.5, 0.0, 0.5, 1.0, 2.0], B)
    table["linear_damping"] = rng.uniform(0.0, 3.0, B); table["angular_damping"] = rng.uniform(0.0, 3.0, B)
    dt, g, d = F(1.0 / 120.0), F(9.82), F(0.25)
    v0, w0 = st.momentum["velocity"].astype(np.float64), st.momentum["angular_velocity"].astype(np.float64)
    active = np.arange(1, B)
    apply_stage(st, table, active, dt, g, d)
    dt64 = float(dt)
    for i in active:
        lin = 1.0 - dt64 * (float(d) + float(table["linear_damping"][i]))
        ang = 1.0 - dt64 * (float(d) + float(table["angular_damping"][i]))
        want = v0[i].copy(); want[1] -= float(g) * dt64 * float(table["gravity_scale"][i])
        _close(st.momentum["velocity"][i], want * lin, rel=2e-6)
        _close(st.momentum["angular_velocity"][i], w0[i] * ang, rel=2e-6)
    # several steps of pure free fall at gravity scale s: v = -s g t (no damping, zero start)
    st.momentum["velocity"][:] = 0
    table["linear_damping"] = 0
    for _ in range(50):
        apply_stage(st, table, active, dt, g, F(0.0))
    _close(st.momentum["velocity"][active, 1], -table["gravity_scale"][active].astype(np.float64) * float(g) * 50 * dt64, rel=1e-5)


def test_torque_gives_the_world_inverse_inertia_times_torque_on_rotated_boxes():
    st, rng = _state(200, 6)
    B = st.scene.n_bodies
    table = default_table(B)
    table["torque"] = rng.normal(0.0, 3.0, (B, 3)); table["force"] = rng.normal(0.0, 3.0, (B, 3))
    dt = F(1.0 / 60.0)
    st.momentum["velocity"] = 0; st.momentum["angular_velocity"] = 0   # the change alone, without the cancellation of a float32 difference
    v0, w0 = st.momentum["velocity"].astype(np.float64), st.momentum["angular_velocity"].astype(np.float64)
    active = np.arange(1, B)
    pushed = apply_stage(st, table, active, dt, F(0.0), F(0.0))
    assert np.array_equal(np.sort(pushed), active) and (st.idle[active] == 0).all()
    for i in active:
        R = _quat_matrix64(st.transforms["rotation"][i].astype(np.float64))
        Iw = R @ np.diag(st.properties["inertia_inverse"][i].astype(np.float64)) @ R.T
        _close(st.momentum["angular_velocity"][i] - w0[i], Iw @ table["torque"][i].astype(np.float64) * float(dt), rel=3e-5)
        _close(st.momentum["velocity"][i] - v0[i], float(st.properties["mass_inverse"][i]) * table["force"][i].astype(np.float64) * float(dt), rel=3e-5)


def test_a_body_frame_force_turns_with_the_body():
    st, rng = _state(100, 7)
    B = st.scene.n_bodies
    table = default_table(B)
    table["flags"] = scenes.BODY_FORCE_LOCAL
    table["force"] = (0.0, 5.0, 0.0); table["torque"] = (0.0, 0.0, 2.0)
    local = rng.normal(0.0, 1.0, (B, 3)).astype(F)
    q = st.transforms["rotation"].astype(np.float64)
    for i in range(1, B):   # qrot is R r
        _close(qrot(st.transforms["rotation"][i:i + 1], local[i:i + 1])[0], _quat_matrix64(q[i]) @ local[i].astype(np.float64), rel=1e-5)
    st.momentum["velocity"] = 0
    v0 = st.momentum["velocity"].astype(np.float64)
    dt = F(0.01)
    apply_stage(st, table, np.arange(1, B), dt, F(0.0), F(0.0))
    for i in range(1, B):
        thrust = _quat_matrix64(q[i]) @ np.array([0.0, 5.0, 0.0])   # the body's own up axis in the world
        _close(st.momentum["velocity"][i] - v0[i], float(st.properties["mass_inverse"][i]) * thrust * float(dt), rel=3e-5)
    # a quarter turn about z: body up (0, 1, 0) points along world -x
    s2 = np.sqrt(F(0.5))
    f = qrot(np.array([[0.0, 0.0, s2, s2]], F), np.array([[0.0, 5.0, 0.0]], F))[0]
    assert abs(f[0] + 5.0) < 1e-5 and abs(f[1]) < 1e-5 and f[2] == 0


def test_remove_and_add_move_the_table_rows_with_their_bodies():
    t = default_table(8)
    t["gravity_scale"] = np.arange(8, dtype=F)
    r = remove_table(t, [2, 5])
    assert r["body"].tolist() == list(range(6)) and r["gravity_scale"].tolist() == [0, 1, 3, 4, 6, 7]
    a = add_table(r, 3)
    assert a["body"].tolist() == list(range(9)) and a["gravity_scale"][6:].tolist() == [1, 1, 1]


def test_sleep_rules_on_a_settling_pile():
    s, pile_a, pile_b = two_piles()
    # gravity scale 0.5 on every body: the piles still fall asleep
    o = BodyForceOracleSim(s)
    half = scenes.default_body_forces(np.arange(1, s.n_bodies)); half["gravity_scale"] = 0.5
    o.set_body_forces(half)
    for _ in range(1200):
        o.step()
        if o.active.count == 0:
            break
    assert o.active.count == 0, "a pile at gravity scale 0.5 never fell asleep"
    # a constant downward force on the bottom box of pile a: its island never sleeps, pile b does
    o = BodyForceOracleSim(s)
    for _ in range(1200):
        o.step()
        if o.active.count == 0:
            break
    assert o.active.count == 0
    press = scenes.default_body_forces([pile_a[0]]); press["force"] = (0.0, -20.0, 0.0)
    o.set_body_forces(press)
    for _ in range(400):
        o.step()
        got = set(o.active_indices[:o.active.count].tolist())
        assert set(pile_a.tolist()) <= got and not (got & set(pile_b.tolist()))
    # cleared (force 0): the island falls asleep again
    o.set_body_forces(scenes.default_body_forces([pile_a[0]]))
    for _ in range(1200):
        o.step()
        if o.active.count == 0:
            break
    assert o.active.count == 0, "the island did not sleep after its force was cleared"
