"""Body impulses on the device (nb_apply_body_impulses, nb_apply_radial_impulse; DESIGN.md section 8.9) against the host edit they replace:
a twin context edited through download_bodies -> tests/impulse_ref.py -> upload_bodies stays byte-identical through a run that sleeps and
wakes (edits between steps and between nb_collide and nb_setup_contact_constraints); the oracle at every stage with the restated edit;
the restated world inverse inertia against the device's; the wake scope of a hit; the explosion's hit set; graph replay against plain
launches; ordering after nb_upload_bodies; throughput mode; and the argument errors."""
import ctypes
import types
import numpy as np
import pytest
import nudge_b200
from nudge_b200 import scenes
from tests.impulse_ref import apply_body_impulses, apply_radial_impulse, radial_hits, random_impulses, world_inverse_inertia
from tests.parity_util import Report, compare_oracle_gpu_step
from tests.gpu_util import side_stream
from tests.test_body_impulse_oracle import two_piles, settle_and_sleep

pytestmark = pytest.mark.gpu
NB_ERR_ARGUMENT = -3


def _state(x):
    x.download_bodies(); x.download_contacts(); x.download_cache()
    c = x.contacts_view()
    parts = [x.transforms, x.momentum, x.idle, c["data"], c["bodies"], c["tags"], c["features"], c["sleeping"], c["active"]]
    cv = x.cache_view()
    return b"".join(np.ascontiguousarray(a).tobytes() for a in parts + [cv["tags"], cv["features"], cv["data"]])


def _counts(x):
    c = x.counts()
    return (c.pairs, c.live_pairs, c.contacts, c.sleeping, c.active, c.cache, c.culled, c.batches, c.levels, c.overflow)


def _bodies(x):
    x.download_bodies()
    return x.transforms.tobytes() + x.momentum.tobytes() + x.idle.tobytes()


def _host_copy(x):
    """The downloaded body rows of `x` as a restatement target."""
    x.download_bodies()
    return types.SimpleNamespace(transforms=x.transforms.copy(), properties=x.properties.copy(), momentum=x.momentum.copy(), idle=x.idle.copy())


def _mixed_scene(seed):
    s = scenes.demo_scene(150, 150, iterations=4, spread=6.0, height=8.0, seed=seed)
    s.transforms["rotation"][1:] = scenes._random_unit_quaternions(np.random.default_rng(seed), s.n_bodies - 1)
    return s


def _edits(rng, i, B):
    """The edits of step i: an impulse list (duplicates, zero impulses, off-centre offsets) on some steps, a radial impulse on others."""
    rows = radial = None
    if i % 3 == 0:
        pool = rng.integers(1, B, 6) if i % 2 else np.arange(1, B)
        rows = random_impulses(rng, pool, int(rng.integers(1, 40)))
    if i % 7 == 2:
        radial = (rng.uniform(-4.0, 4.0, 3).astype(np.float32) + np.float32([0.0, 2.0, 0.0]),np.float32(rng.uniform(2.0, 6.0)), np.float32(rng.uniform(-10.0, 20.0)))
    return rows, radial


def _edit_both(dev, twin, rows, radial, kinematic=()):
    if rows is not None:
        dev.apply_body_impulses(rows)
    if radial is not None:
        dev.apply_radial_impulse(*radial)
    if rows is None and radial is None:
        return
    twin.download_bodies()
    if rows is not None:
        apply_body_impulses(twin, rows)
    if radial is not None:
        apply_radial_impulse(twin, *radial, kinematic=kinematic)
    twin.upload_bodies()


def _rest_of_step(x):
    x.apply_gravity_damping(); x.read_cached_impulses(); x.setup_contact_constraints(); x.apply_impulses(int(x.scene.iterations))
    x.update_cached_impulses(); x.write_cached_impulses(); x.advance()


@pytest.mark.parametrize("where", ["between_steps", "after_collide"])
def test_device_edit_equals_the_host_round_trip_bit_for_bit(where):
    s = _mixed_scene(11)
    dev, twin = nudge_b200.Sim(s, stream=side_stream()), nudge_b200.Sim(s, stream=side_stream())
    rng = np.random.default_rng(21)
    sleeping = woken = 0
    for i in range(72):
        if i == 30:   # put most of the scene to sleep, identically in both
            asleep = np.random.default_rng(5).random(s.n_bodies) < 0.8
            for x in (dev, twin):
                x.download_bodies(); x.idle[asleep] = 0xff
                x.momentum["velocity"][asleep] = 0; x.momentum["angular_velocity"][asleep] = 0
                x.upload_bodies()
        rows, radial = _edits(rng, i, s.n_bodies)
        if where == "between_steps":
            _edit_both(dev, twin, rows, radial)
            dev.step(); twin.step()
        else:
            dev.collide(); twin.collide()
            _edit_both(dev, twin, rows, radial)
            _rest_of_step(dev); _rest_of_step(twin)
        assert _state(dev) == _state(twin), (where, i)
        cd = _counts(dev)
        assert cd == _counts(twin), (where, i)
        sleeping += cd[3]
        if i > 30 and rows is not None:
            woken += int((dev.idle[rows["body"]] != 0xff).sum())
    assert sleeping > 0 and woken > 0


def test_restated_edit_on_the_oracle_equals_the_device_at_every_stage():
    from oracle import pyoracle
    s = scenes.box_drop(1500, iterations=8)
    o = pyoracle.OracleSim(s)
    g = nudge_b200.Sim(s, contact_capacity=o.cap, debug=True)
    rng = np.random.default_rng(4)
    B = s.n_bodies
    for i in range(14):
        edited = False
        if i in (3, 6, 9, 12):
            rows = random_impulses(rng, rng.integers(1, B, 30) if i == 9 else np.arange(1, B), 25)
            g.apply_body_impulses(rows); apply_body_impulses(o, rows)
            edited = True
        if i in (5, 10):
            c = s.transforms["position"][1:].mean(0)
            g.apply_radial_impulse(c, 6.0, 20.0 if i == 5 else -8.0); apply_radial_impulse(o, c, 6.0, 20.0 if i == 5 else -8.0)
            edited = True
        if edited:
            g.download_bodies()
            assert g.momentum.tobytes() == o.momentum.tobytes() and g.idle.tobytes() == o.idle.tobytes(), i
        rep = Report("step %d" % i)
        assert compare_oracle_gpu_step(o, g, rep), str(rep)


def test_restated_world_inverse_inertia_equals_the_device_buffer():
    g = nudge_b200.Sim(_mixed_scene(4))
    for _ in range(5):
        g.step_staged()
    g.collide(); g.apply_gravity_damping(); g.read_cached_impulses(); g.setup_contact_constraints()
    g.download_bodies()
    dev = g.debug("inertia", np.float32).reshape(-1, 8)
    W = world_inverse_inertia(g.transforms["rotation"], g.properties)
    assert np.ascontiguousarray(dev[:, [0, 1, 2, 4, 5, 6]]).tobytes() == W.tobytes()


def test_a_hit_wakes_exactly_its_island_and_leaves_the_other_pile_alone():
    s, pile_a, pile_b = two_piles()
    g = nudge_b200.Sim(s, stream=side_stream())
    settle_and_sleep(g)
    g.collide(); g.download_contacts()
    assert g.counts().active == 0
    _rest_of_step(g)
    g.download_bodies()
    before_b = (g.transforms[pile_b].tobytes(), g.momentum[pile_b].tobytes(), g.idle[pile_b].tobytes())
    hit = np.zeros(1, scenes.BODY_IMPULSE)
    hit["body"] = pile_a[2]; hit["impulse"] = (0.5, 0.0, 0.0); hit["offset"] = (0.0, 0.3, 0.0)
    g.apply_body_impulses(hit)
    g.collide(); g.download_contacts()
    assert g.counts().active == len(pile_a)
    assert np.array_equal(np.sort(g.contacts_view()["active"]), np.sort(pile_a))
    _rest_of_step(g)
    for _ in range(10):
        g.step()
    g.download_bodies()
    assert (g.transforms[pile_b].tobytes(), g.momentum[pile_b].tobytes(), g.idle[pile_b].tobytes()) == before_b


def test_explosion_hits_exactly_the_restated_bodies():
    s = _mixed_scene(12)
    center = np.float32([0.0, 2.0, 0.0])
    kb = 1 + int(np.argmin(np.linalg.norm(s.transforms["position"][1:] - center, axis=1)))
    s.kinematic = np.array([(kb, (0.0, 0.0, 0.0), (0.0, 0.0, 0.0), 0)], scenes.KINEMATIC)
    g = nudge_b200.Sim(s, stream=side_stream())
    for _ in range(20):
        g.step()
    radius = np.float32(5.0)
    for impulse in (12.0, -5.0, 0.0):
        want = _host_copy(g)
        before = want.momentum.copy(), want.idle.copy()
        hit = apply_radial_impulse(want, center, radius, impulse, kinematic=[kb])
        g.apply_radial_impulse(center, radius, impulse)
        g.download_bodies()
        assert g.momentum.tobytes() == want.momentum.tobytes() and g.idle.tobytes() == want.idle.tobytes(), impulse
        inside, _, dist = radial_hits(want, center, radius)
        assert hit.sum() > 10 and (~hit).sum() > 10 and dist[kb] < radius and inside.sum() == hit.sum() + 1
        keep = ~hit
        assert keep[0] and keep[kb] and np.linalg.norm(want.transforms["position"][0] - center) < radius   # body 0 and the kinematic body: inside, untouched
        assert g.momentum[keep].tobytes() == before[0][keep].tobytes() and g.idle[keep].tobytes() == before[1][keep].tobytes()
        assert (g.idle[hit] == 0).all()
        if impulse == 0.0:   # only wakes: every velocity keeps its value (a -0.0 component may become +0.0)
            assert np.array_equal(g.momentum["velocity"], before[0]["velocity"]) and np.array_equal(g.momentum["angular_velocity"], before[0]["angular_velocity"])
        else:
            assert not np.array_equal(g.momentum["velocity"][hit], before[0]["velocity"][hit])
        g.step()


def test_graph_replay_with_edits_every_step_equals_plain_launches():
    s = _mixed_scene(13)
    a, p = nudge_b200.Sim(s, stream=side_stream()), nudge_b200.Sim(s)   # p: the legacy default stream, plain launches
    a.step(); p.step()
    rng = np.random.default_rng(8)
    for i in range(25):
        rows = random_impulses(rng, np.arange(1, s.n_bodies), 12)
        c0 = a.launch_count()
        a.apply_body_impulses(rows); p.apply_body_impulses(rows)
        c1 = a.launch_count()
        assert c1 - c0 == 3, i
        if i % 2:
            a.apply_radial_impulse((0.0, -6.0, 0.0), 5.0, 9.0); p.apply_radial_impulse((0.0, -6.0, 0.0), 5.0, 9.0)
        c2 = a.launch_count()
        assert c2 - c1 == (1 if i % 2 else 0), i
        a.step(); p.step()
        assert a.launch_count() - c2 == 61, i
        assert _state(a) == _state(p), i
    assert a.debug_scalar("graph_active") == 1


def test_a_call_right_after_upload_bodies_sees_the_uploaded_rows():
    s = _mixed_scene(14)
    g = nudge_b200.Sim(s, stream=side_stream())
    for _ in range(5):
        g.step()
    rng = np.random.default_rng(9)
    B = s.n_bodies
    small = random_impulses(rng, np.arange(1, B), 5)
    g.apply_body_impulses(small)   # the staging buffers then grow for the long list below
    g.download_bodies()
    g.momentum["velocity"][1:] += np.float32(1.0); g.momentum["angular_velocity"][1:] -= np.float32(0.5); g.idle[1:] = 7
    want = types.SimpleNamespace(transforms=g.transforms.copy(), properties=g.properties.copy(), momentum=g.momentum.copy(), idle=g.idle.copy())
    rows = np.concatenate([random_impulses(rng, rng.integers(1, B, 40), 3000), random_impulses(rng, np.arange(1, B), B - 1, duplicates=False)])
    rows = rows[rng.permutation(len(rows))]
    apply_body_impulses(want, rows)
    g.upload_bodies()
    g.apply_body_impulses(rows)
    g.download_bodies()
    assert g.momentum.tobytes() == want.momentum.tobytes() and g.idle.tobytes() == want.idle.tobytes()


def test_throughput_mode_edit_equals_the_restatement_and_the_step_runs():
    s = _mixed_scene(15)
    g = nudge_b200.Sim(s, stream=side_stream())
    g.set_solver_mode("throughput")
    for _ in range(10):
        g.step()
    rng = np.random.default_rng(10)
    rows = random_impulses(rng, np.arange(1, s.n_bodies), 50)
    want = _host_copy(g)
    apply_body_impulses(want, rows); apply_radial_impulse(want, (0.0, -6.0, 0.0), 4.0, 10.0)
    g.apply_body_impulses(rows); g.apply_radial_impulse((0.0, -6.0, 0.0), 4.0, 10.0)
    g.download_bodies()
    assert g.momentum.tobytes() == want.momentum.tobytes() and g.idle.tobytes() == want.idle.tobytes()
    for _ in range(3):
        g.step()
    c = g.counts()
    g.download_bodies()
    assert c.overflow == 0 and c.contacts > 0 and np.isfinite(g.transforms["position"]).all()


def test_argument_errors_change_nothing():
    s = _mixed_scene(16)
    s.kinematic = np.array([(7, (0.0, 0.1, 0.0), (0.0, 0.0, 0.0), 0)], scenes.KINEMATIC)
    g = nudge_b200.Sim(s)
    g.step_staged()
    before = _bodies(g)
    good = random_impulses(np.random.default_rng(1), np.arange(8, 40), 4)
    for bad_body in (0, s.n_bodies, 7):
        bad = np.concatenate([good, good[:1]]); bad["body"][-1] = bad_body
        bad = np.ascontiguousarray(bad)
        assert g.lib.nb_apply_body_impulses(g.ctx, bad.ctypes.data_as(ctypes.c_void_p), len(bad), g.stream) == NB_ERR_ARGUMENT, bad_body
    assert g.lib.nb_apply_body_impulses(g.ctx, None, 3, g.stream) == NB_ERR_ARGUMENT
    assert g.lib.nb_apply_body_impulses(g.ctx, None, 0, g.stream) == 0
    for radius in (0.0, -1.0, float("nan"), float("inf")):
        e = np.zeros(1, scenes.RADIAL_IMPULSE); e["radius"] = radius; e["impulse"] = 5.0
        assert g.lib.nb_apply_radial_impulse(g.ctx, e.ctypes.data_as(ctypes.c_void_p), g.stream) == NB_ERR_ARGUMENT, radius
    assert g.lib.nb_apply_radial_impulse(g.ctx, None, g.stream) == NB_ERR_ARGUMENT
    assert _bodies(g) == before
    with pytest.raises(nudge_b200.NudgeError, match="kinematic"):
        g.apply_body_impulses(np.array([(7, (0, 0, 0), (1, 0, 0), (0, 0, 0), (0, 0))], scenes.BODY_IMPULSE))
