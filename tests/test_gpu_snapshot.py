"""Device-resident snapshots (nb_snapshot_save / nb_snapshot_restore; DESIGN.md section 8.12): a rollback over steps that carry impulses,
kinematic velocities, force edits, a spawn and a despawn re-simulates byte for byte (state file, user rows, sensor overlaps and drained
events); restores across structural changes equal a twin loaded from the saved state file; saving changes nothing, costs one launch and can
be captured into an application's CUDA graph; nb_step's graph is kept or re-recorded by the stated rule; throughput mode; the refusals."""
import os
import tempfile
import numpy as np
import pytest
import nudge_b200
from nudge_b200 import scenes, ROW
from tests.gpu_util import side_stream
from tests.test_body_impulse_oracle import two_piles, settle_and_sleep

pytestmark = pytest.mark.gpu
NB_ERR_ARGUMENT = -3
TOL = 1e-4                       # throughput mode's run-to-run tolerance, of the velocity scale (tests/test_gpu_throughput.py)
SENSOR_PAIRS = 4096
SPARE = 200
KIN = 7                          # the moving platform
JOINED = list(range(20, 29))     # a chain of ball joints over these bodies


def _saved(x):
    with tempfile.TemporaryDirectory() as d:
        p = os.path.join(d, "s.nbstate")
        x.save_state(p)
        return open(p, "rb").read()


def _ball_rows(pairs):
    """Three point-to-point rows (x, y, z) per joined pair."""
    rows = np.zeros(3 * len(pairs), ROW)
    for j, (a, b) in enumerate(pairs):
        for k in range(3):
            r = rows[3 * j + k]
            r["a"], r["b"] = a, b
            r["lin_a"][k], r["lin_b"][k] = 1.0, -1.0
            r["lo"], r["hi"] = -np.inf, np.inf
    return rows


def _scene(seed=5):
    """About 1,500 bodies falling on the ground, sparse enough to stay within the contact capacity (a step that overflows it is undefined): a sensor zone on body 0, a filter table with NB_FILTER_SKIP_CONNECTED over connections, a kinematic
    platform, a chain of ball joints (connected, so their islands join) and a body force table."""
    rng = np.random.default_rng(seed)
    s = scenes.demo_scene(750, 750, iterations=4, spread=20.0, height=60.0, seed=seed)
    nb = s.n_boxes
    z = np.zeros(1, scenes.TRANSFORM); z["rotation"][:, 3] = 1; z["position"] = (0.0, 0.0, 0.0)
    zb = np.zeros(1, scenes.BOX); zb["size"] = (6.0, 8.0, 6.0)
    s.box_tags = np.concatenate([s.box_tags, [int(max(s.box_tags.max(), s.sphere_tags.max())) + 1]]).astype(np.uint32)
    s.box_data = np.concatenate([s.box_data, zb]); s.box_transforms = np.concatenate([s.box_transforms, z])
    K = s.n_colliders
    s.sensors = np.zeros(K, np.uint8); s.sensors[nb] = 1
    s.collision_filters = np.zeros(K, scenes.FILTER)
    s.collision_filters["category"] = 1 << rng.integers(0, 3, K)
    s.collision_filters["mask"] = 0xffff
    s.filter_flags = scenes.FILTER_SKIP_CONNECTED
    s.kinematic = np.array([(KIN, (0.0, 0.0, 0.0), (0.0, 0.0, 0.0), 0)], scenes.KINEMATIC)
    s.transforms["position"][KIN] = (0.0, -9.0, 0.0)
    pairs = list(zip(JOINED[:-1], JOINED[1:]))
    s.connections = np.array(pairs + [(60, 61), (70, 80)], scenes.PAIR32)
    f = scenes.default_body_forces(np.arange(100, 140))
    f["gravity_scale"] = rng.uniform(0.0, 2.0, len(f)).astype(np.float32)
    s.body_forces = f
    return s, _ball_rows(pairs)


def _sim(s, rows, stream=None):
    x = nudge_b200.Sim(s, stream=side_stream() if stream is None else stream, max_bodies=s.n_bodies + SPARE, max_boxes=s.n_boxes + SPARE,
                       max_spheres=s.n_spheres + SPARE, contact_capacity=48 * (s.n_bodies + SPARE))
    x.upload_sensors(s.sensors, SENSOR_PAIRS)
    x.upload_constraint_rows(rows)
    return x


def _filters(n):
    f = np.zeros(n, scenes.FILTER)
    f["category"], f["mask"] = 1, 0xffff
    return f


def _fragment(rng, n, first_tag):
    """n boxes dropped beside the pile."""
    return scenes.fragment(rng.uniform(-3, 3, (n, 3)) + (20, 0, 0), "box", rng.uniform(0.3, 0.7, (n, 3)), first_tag)


def _inputs(x, i):
    """The application's inputs before step i, a function of i and the scene alone: a few impulses, the platform's velocity, force edits,
    a spawn at step 35 and a despawn at step 37."""
    rng = np.random.default_rng(1000 + i)
    B = x.scene.n_bodies
    pool = np.setdiff1d(np.arange(1, B), [KIN] + JOINED + list(range(100, 140)))
    hits = np.zeros(3, scenes.BODY_IMPULSE)
    hits["body"] = rng.choice(pool, 3, replace=False)
    hits["impulse"] = rng.uniform(-0.5, 0.5, (3, 3)).astype(np.float32)
    x.apply_body_impulses(hits)
    w = float(np.sin(0.2 * i))
    x.upload_kinematic_bodies(np.array([(KIN, (w, 0.0, 0.0), (0.0, 0.1 * w, 0.0), 0)], scenes.KINEMATIC))
    f = scenes.default_body_forces(rng.choice(np.arange(100, 140), 4, replace=False))
    f["gravity_scale"] = rng.uniform(0.0, 2.0, 4).astype(np.float32)
    f["force"] = rng.uniform(-1.0, 1.0, (4, 3)).astype(np.float32)
    x.set_body_forces(f)
    if i == 35:
        fr = _fragment(rng, 6, 500000)
        x.add_bodies(fr, filters=_filters(fr.n_colliders), sensors=np.zeros(fr.n_colliders, np.uint8))
    if i == 37:
        x.remove_bodies(np.sort(rng.choice(pool[pool > 140], 5, replace=False)))   # the platform, joints and forced bodies keep their indices


def _events(x):
    return x.contact_events()[0].tobytes()


def test_rollback_re_simulates_byte_for_byte():
    s, rows = _scene()
    x = _sim(s, rows)
    x.enable_contact_events(1 << 16)
    ring = [nudge_b200.Snapshot(x) for _ in range(8)]
    files, events, nrows = {}, {}, len(rows)
    for i in range(40):
        x.snapshot(into=ring[i % 8])
        if i >= 32:
            files[i] = _saved(x)
        _inputs(x, i)
        x.step()
        events[i] = _events(x)
    final, final_rows, final_ov = _saved(x), x.download_constraint_rows(nrows), x.sensor_overlaps()
    assert len(final_ov) > 0 and sum(len(e) for e in events.values()) > 0
    assert x.debug_scalar("graph_active") == 1 and x.counts().overflow == 0
    x.restore(ring[33 % 8])
    assert _saved(x) == files[33]
    for i in range(33, 40):
        _inputs(x, i)
        x.step()
        assert _events(x) == events[i], i   # step numbers included
    assert _saved(x) == final
    assert np.array_equal(x.download_constraint_rows(nrows), final_rows)
    assert x.sensor_overlaps().tobytes() == final_ov.tobytes()
    for k in (38, 34, 39, 32, 36, 33, 35, 37):   # out of order, across the spawn and the despawn
        x.restore(ring[k % 8])
        assert _saved(x) == files[k], k
        assert x.scene.n_bodies == (s.n_bodies + (6 if k > 35 else 0) - (5 if k > 37 else 0)), k


def test_restore_across_structural_changes_equals_a_loaded_twin():
    s, rows = _scene(9)
    s.body_forces = None
    x = _sim(s, rows)
    saved = []

    def keep():
        saved.append((x.snapshot(), _saved(x), x.download_constraint_rows(len(rows))))

    for _ in range(5):
        x.step()
    keep()                                          # a kinematic set, no force table, before the spawn
    x.upload_kinematic_bodies(None)
    x.step()
    keep()                                          # no kinematic set, no force table
    f = scenes.default_body_forces(np.arange(100, 110)); f["gravity_scale"] = 0.25
    x.set_body_forces(f)
    x.step()
    keep()                                          # a force table, before the spawn
    x.add_bodies(_fragment(np.random.default_rng(1), 8, 600000), filters=_filters(8), sensors=np.zeros(8, np.uint8))
    x.upload_constraint_rows(rows[:6])              # rows that differ
    for _ in range(3):
        x.step()
    for snap, file, saved_rows in reversed(saved):
        x.restore(snap)
        assert _saved(x) == file
        twin = _sim(s, rows)
        with tempfile.TemporaryDirectory() as d:
            p = os.path.join(d, "s.nbstate")
            open(p, "wb").write(file)
            twin.load_state(p)
        twin.upload_constraint_rows(saved_rows)
        for i in range(20):
            x.step(); twin.step()
            assert _saved(x) == _saved(twin), i
        assert np.array_equal(x.download_constraint_rows(len(saved_rows)), twin.download_constraint_rows(len(saved_rows)))
        twin.close()


def _sleep_wake_run(x, save):
    snap = nudge_b200.Snapshot(x)
    per_save = []
    settle_and_sleep(x, 30)
    for i in range(60):
        if i == 25:
            x.apply_radial_impulse((0.0, 0.0, 0.0), 3.0, 0.5)
        if save:
            n = x.launch_count()
            x.snapshot(into=snap)
            per_save.append(x.launch_count() - n)
        x.step()
    return _saved(x), per_save, snap


def test_save_changes_nothing_costs_one_launch_and_can_be_captured():
    import torch
    s, _, _ = two_piles()
    a, b = nudge_b200.Sim(s, stream=side_stream()), nudge_b200.Sim(s, stream=side_stream())
    fa, per_save, snap = _sleep_wake_run(a, True)
    fb, _, _ = _sleep_wake_run(b, False)
    assert fa == fb
    assert per_save == [1] * 60
    n = a.launch_count()
    a.restore(snap)
    assert a.launch_count() - n == 1
    # a save captured into the application's graph on a side stream, replayed later
    st = torch.cuda.Stream()
    c = nudge_b200.Sim(s, stream=st.cuda_stream)
    for _ in range(5):
        c.step()
    snap = c.snapshot()   # sizes the snapshot
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=st):
        c.snapshot(into=snap)
    for _ in range(4):
        c.step()
    with torch.cuda.stream(st):
        g.replay()
    want = _saved(c)
    for _ in range(6):
        c.step()
    c.restore(snap)
    assert _saved(c) == want


def test_graph_is_kept_unless_the_step_changes():
    s, rows = _scene(13)
    x = _sim(s, rows)
    for _ in range(3):
        x.step()
    rec = lambda: x.debug_scalar("graph_records")
    snap = x.snapshot()
    for _ in range(3):
        x.step()
    n = rec()
    x.restore(snap); x.step()
    assert rec() == n and x.debug_scalar("graph_active") == 1
    x.add_bodies(_fragment(np.random.default_rng(2), 5, 700000), filters=_filters(5), sensors=np.zeros(5, np.uint8))
    x.step()
    n = rec()
    x.restore(snap); x.step()
    assert rec() == n + 1
    x.clear_body_forces(); x.step()
    n = rec()
    x.restore(snap); x.step(); x.step()
    assert rec() == n + 1


def test_throughput_mode_restore_is_byte_exact():
    s, rows = _scene(17)
    x = _sim(s, rows)
    x.set_solver_mode("throughput")
    for _ in range(10):
        x.step()
    snap = x.snapshot()
    want = _saved(x)
    after = []
    for _ in range(5):
        x.step(); x.download_bodies(); after.append(x.momentum.copy())
    x.restore(snap)
    assert _saved(x) == want and x.solver_mode() == "throughput"
    scale = max(1.0, float(np.abs(after[0]["velocity"]).max()))
    for k in range(5):
        x.step(); x.download_bodies()
        for f in ("velocity", "angular_velocity"):
            assert np.abs(x.momentum[f].astype(np.float64) - after[k][f]).max() < TOL * scale, (k, f)


def test_refusals_change_nothing():
    s, rows = _scene(21)
    x, y = _sim(s, rows), _sim(s, rows)
    for _ in range(3):
        x.step(); y.step()
    L, ctx, st = x.lib, x.ctx, x.stream
    fresh = nudge_b200.Snapshot(x)
    before = _saved(x)
    assert L.nb_snapshot_restore(ctx, fresh.handle, st) == NB_ERR_ARGUMENT       # never saved
    other = y.snapshot()
    assert L.nb_snapshot_save(ctx, other.handle, st) == NB_ERR_ARGUMENT          # another context's
    assert L.nb_snapshot_restore(ctx, other.handle, st) == NB_ERR_ARGUMENT
    x.collide()
    assert L.nb_snapshot_save(ctx, fresh.handle, st) == NB_ERR_ARGUMENT          # between nb_collide and nb_advance
    assert L.nb_snapshot_restore(ctx, fresh.handle, st) == NB_ERR_ARGUMENT       # still never saved
    x.apply_gravity_damping(); x.read_cached_impulses(); x.setup_contact_constraints(); x.apply_impulses(4)
    x.update_cached_impulses(); x.write_cached_impulses(); x.advance()
    y.step_staged()
    assert _saved(x) == _saved(y) != before
    x.snapshot(into=fresh)   # legal again after nb_advance
    z = _sim(s, rows)
    zs = z.snapshot()
    z.shard_create(0, 1, None, 16, 16)
    zf = _saved(z)
    assert z.lib.nb_snapshot_save(z.ctx, zs.handle, z.stream) == NB_ERR_ARGUMENT
    assert z.lib.nb_snapshot_restore(z.ctx, zs.handle, z.stream) == NB_ERR_ARGUMENT
    assert _saved(z) == zf
    with pytest.raises(nudge_b200.NudgeError):
        nudge_b200.Snapshot(z)
    z.close()
    zs.close()   # its context freed it
