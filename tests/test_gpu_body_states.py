"""Body states on the device (nb_get_body_states, nb_set_body_states; DESIGN.md section 8.19) against the host read and edit they replace:
the gather equals nb_download_bodies' rows; a set equals tests/body_state_ref.py's edit sent through nb_upload_bodies, byte for byte in the
state file right after the edit and through 60 further steps of a scene with every table an edit must leave alone; throughput mode; a
teleported bottom crate wakes the sleeping stack above it (and without the wake the stack floats); device pointers with invalid entries;
a torch CUDA graph of get -> torch op -> set against the same calls uncaptured; the step graph and the launches per step kept; snapshots;
and the refusals.  The launch counts against torch.profiler are in test_gpu_launch_count_body_states.py."""
import ctypes
import os
import tempfile
import numpy as np
import pytest
import torch
import nudge_b200
from nudge_b200 import abi, scenes
from tests.body_state_ref import REMOVED, get_states, set_states, valid
from tests.spawn_ref import live_scene
from tests.gpu_util import side_stream
from tests.test_body_impulse_oracle import two_piles, settle_and_sleep
from tests.test_gpu_joints import _at_rest

pytestmark = pytest.mark.gpu
NB_ERR_ARGUMENT = -3
POSE, VEL = abi.BODY_POSE, abi.BODY_VELOCITY
SENSOR_PAIRS = 4096


def _saved(x):
    with tempfile.TemporaryDirectory() as d:
        p = os.path.join(d, "s.nbstate")
        x.save_state(p)
        return open(p, "rb").read()


def _kin(x):
    return [] if x.scene.kinematic is None else x.scene.kinematic["body"].tolist()


def _scene(seed=41):
    """Boxes and spheres on the ground, three sensor zones on body 0, a filter table with NB_FILTER_SKIP_CONNECTED and connections, a
    kinematic platform (body 7), a body force table; ball joints are uploaded by _sim."""
    rng = np.random.default_rng(seed)
    s = scenes.demo_scene(150, 150, iterations=4, spread=6.0, height=8.0, seed=seed)
    nb = s.n_boxes
    tags0 = int(max(s.box_tags.max(), s.sphere_tags.max())) + 1
    z = np.zeros(3, scenes.TRANSFORM); z["rotation"][:, 3] = 1; z["position"] = [(-3.0, 4.0, 0.0), (3.0, 4.0, 2.0), (0.0, 4.0, -3.0)]
    zb = np.zeros(3, scenes.BOX); zb["size"] = (2.0, 4.0, 2.0)
    s.box_tags = np.concatenate([s.box_tags, tags0 + np.arange(3, dtype=np.uint32)])
    s.box_data = np.concatenate([s.box_data, zb]); s.box_transforms = np.concatenate([s.box_transforms, z])
    K = s.n_colliders
    s.sensors = np.zeros(K, np.uint8); s.sensors[nb:nb + 3] = 1
    s.collision_filters = np.zeros(K, scenes.FILTER)
    s.collision_filters["category"] = 1 << rng.integers(0, 3, K)
    s.collision_filters["mask"] = 0xffff
    s.filter_flags = scenes.FILTER_SKIP_CONNECTED
    s.kinematic = np.array([(7, (0.0, 0.0, 0.0), (0.0, 0.0, 0.0), 0)], scenes.KINEMATIC)
    s.transforms["position"][7] = (0.0, -9.0, 0.0)
    s.connections = np.array([(10, 11), (20, 21), (30, 0), (40, 41), (60, 61), (70, 80)], scenes.PAIR32)
    f = scenes.default_body_forces(np.arange(3, s.n_bodies, 9))
    f["gravity_scale"] = 0.5; f["linear_damping"] = 0.1
    s.body_forces = f
    return s


def _sim(s, stream=None):
    x = nudge_b200.Sim(s, stream=side_stream() if stream is None else stream)
    x.upload_sensors(s.sensors, SENSOR_PAIRS)
    rng = np.random.default_rng(5)
    x.upload_joints(np.array([_at_rest(s.transforms, 0, a, b, rng, mid=True) for a, b in ((10, 11), (40, 41), (90, 91), (100, 0))]))
    return x


def _random_rows(rng, B, n, kinematic=()):
    """n rows on random bodies 1 .. B-1 (with duplicates): poses above the pile, unit rotations, modest velocities."""
    r = np.zeros(n, abi.BODY_STATE)
    r["body"] = rng.integers(1, B, n)
    r["body"][: len(kinematic)] = kinematic
    r["position"] = rng.uniform((-6.0, 0.5, -6.0), (6.0, 10.0, 6.0), (n, 3))
    r["rotation"] = scenes._random_unit_quaternions(rng, n)
    r["velocity"] = rng.normal(0.0, 2.0, (n, 3)); r["angular_velocity"] = rng.normal(0.0, 1.0, (n, 3))
    r["idle_counter"] = 99; r["reserved"] = 7
    return r


def _twin_set(t, rows, fields):
    """The host edit: download, restate, upload every body."""
    t.download_bodies(); t.download_cache()
    new, woken = set_states(live_scene(t), rows, fields, t.cache_view()["tags"], _kin(t))
    t.transforms[:] = new.transforms; t.momentum[:] = new.momentum; t.idle[:] = new.idle
    t.upload_bodies()
    return woken


def _asleep(x):
    x.download_bodies(); x.idle[1:] = 0xff
    x.momentum["velocity"][1:] = 0; x.momentum["angular_velocity"][1:] = 0
    x.upload_bodies()


@pytest.mark.parametrize("device", [False, True])
def test_gather_equals_download_bodies_rows(device):
    s = _scene(42)
    g = _sim(s)
    for _ in range(15):
        g.step()
    B = s.n_bodies
    rng = np.random.default_rng(1)
    lists = [rng.integers(0, B, 500).astype(np.uint32), np.array([0], np.uint32), np.arange(B, dtype=np.uint32)[::-1].copy(), None]
    if device:
        lists += [np.array([3, B, 0xffffffff, 0, B - 1], np.uint32)]
    g.download_bodies()
    live = live_scene(g)
    for idx in lists:
        n = B if idx is None else len(idx)
        want = get_states(live, idx)
        if device:
            ext = B + 5 if idx is None else n   # a null list past the body count: the tail rows are NB_REMOVED_BODY rows
            want = get_states(live, np.arange(ext, dtype=np.uint32)) if idx is None else want
            t_idx = None if idx is None else torch.from_numpy(idx.view(np.int32)).cuda()
            out = torch.full((ext * 16,), -1, dtype=torch.int32, device="cuda")
            torch.cuda.synchronize()
            g.get_body_states(device_ptrs=(0 if t_idx is None else t_idx.data_ptr(), out.data_ptr()), n=ext)
            torch.cuda.synchronize()
            got = out.cpu().numpy().view(abi.BODY_STATE)
        else:
            got = g.get_body_states(idx)
        assert got.tobytes() == want.tobytes()
        if idx is None and device:
            assert (got["body"][B:] == REMOVED).all()
    # the rows are the downloaded rows themselves
    rows = g.get_body_states()
    assert rows["position"].tobytes() == np.ascontiguousarray(g.transforms["position"]).tobytes()
    assert rows["velocity"].tobytes() == np.ascontiguousarray(g.momentum["velocity"]).tobytes()
    assert np.array_equal(rows["idle_counter"], g.idle)


@pytest.mark.parametrize("fields", [POSE, VEL, POSE | VEL])
def test_set_equals_the_host_edit_bit_for_bit_for_60_steps(fields):
    s = _scene(43)
    dev, twin = _sim(s), _sim(s)
    for x in (dev, twin):
        x.enable_contact_events(1 << 16)
        for _ in range(40):
            x.step()
        _asleep(x)
        for _ in range(3):
            x.step()
    assert _saved(dev) == _saved(twin)
    rng = np.random.default_rng(fields)
    rows = _random_rows(rng, s.n_bodies, 300, kinematic=[7])
    assert len(np.unique(rows["body"])) < 300
    assert dev.set_body_states(rows, fields) == 0
    woken = _twin_set(twin, rows, fields)
    assert _saved(dev) == _saved(twin)
    listed = np.unique(rows["body"]).size
    assert woken.sum() > listed - 1 if fields & POSE else woken.sum() == listed - 1   # the kinematic body 7 is listed and never woken
    for i in range(60):
        dev.step(); twin.step()
        assert _saved(dev) == _saved(twin), i
        ed, et = dev.contact_events()[0], twin.contact_events()[0]
        assert ed.tobytes() == et.tobytes(), i


def test_throughput_mode_edit_equals_the_restatement_and_the_step_runs():
    s = _scene(44)
    g = _sim(s)
    g.set_solver_mode("throughput")
    for _ in range(10):
        g.step()
    rows = _random_rows(np.random.default_rng(3), s.n_bodies, 200)
    g.download_bodies(); g.download_cache()
    want, _ = set_states(live_scene(g), rows, POSE | VEL, g.cache_view()["tags"], _kin(g))
    g.set_body_states(rows, POSE | VEL)
    g.download_bodies()
    assert (g.transforms.tobytes(), g.momentum.tobytes(), g.idle.tobytes()) == (want.transforms.tobytes(), want.momentum.tobytes(), want.idle.tobytes())
    for _ in range(3):
        g.step()
    c = g.counts()
    g.download_bodies()
    assert c.overflow == 0 and c.contacts > 0 and np.isfinite(g.transforms["position"]).all()


def _settled_piles():
    s, pile_a, pile_b = two_piles()
    g = nudge_b200.Sim(s, stream=side_stream())
    settle_and_sleep(g)
    g.step()
    g.collide(); g.download_contacts()
    assert g.counts().active == 0
    g.apply_gravity_damping(); g.read_cached_impulses(); g.setup_contact_constraints(); g.apply_impulses(8)
    g.update_cached_impulses(); g.write_cached_impulses(); g.advance()
    return g, pile_a, pile_b


def test_teleporting_the_bottom_crate_wakes_the_stack_above_and_not_the_other_pile():
    g, pile_a, pile_b = _settled_piles()
    raw, _, _ = _settled_piles()   # the same run, given only the raw uploaded pose
    g.download_bodies()
    assert _saved(g) == _saved(raw)
    before_b = g.transforms[pile_b].tobytes()
    top = pile_a[-2]
    top_y = g.transforms["position"][top, 1]
    r = np.zeros(1, abi.BODY_STATE)
    r["body"] = pile_a[0]; r["position"] = (60.0, 0.5, 0.0); r["rotation"] = (0.0, 0.0, 0.0, 1.0)
    g.set_body_states(r, POSE | VEL)
    raw.download_bodies()
    raw.transforms["position"][pile_a[0]] = r["position"][0]; raw.transforms["rotation"][pile_a[0]] = r["rotation"][0]
    raw.momentum["velocity"][pile_a[0]] = 0; raw.momentum["angular_velocity"][pile_a[0]] = 0; raw.idle[pile_a[0]] = 0
    raw.upload_bodies()
    g.download_bodies()
    assert g.idle[pile_a[0]] == 0 and g.idle[pile_a[1]] == 0 and (g.idle[pile_b] == 0xff).all()
    g.collide(); g.download_contacts()
    assert sorted(g.contacts_view()["active"].tolist()) == sorted(pile_a.tolist())
    g.apply_gravity_damping(); g.read_cached_impulses(); g.setup_contact_constraints(); g.apply_impulses(8)
    g.update_cached_impulses(); g.write_cached_impulses(); g.advance()
    for _ in range(90):
        g.step(); raw.step()
    g.download_bodies(); raw.download_bodies()
    assert g.transforms[pile_b].tobytes() == before_b and (g.idle[pile_b] == 0xff).all()
    assert g.transforms["position"][top, 1] < top_y - 0.5        # the stack fell into the gap
    assert raw.transforms["position"][top, 1] == top_y              # without the wake it floats, asleep
    assert (raw.idle[pile_a[1:]] == 0xff).all()


def test_device_pointers_skip_invalid_entries_and_equal_the_host_call_on_the_rest():
    s = _scene(45)
    dev, twin = _sim(s), _sim(s)
    for x in (dev, twin):
        for _ in range(20):
            x.step()
    B = s.n_bodies
    for fields in (POSE, VEL, POSE | VEL):
        rows = _random_rows(np.random.default_rng(10 + fields), B, 120)
        rows["body"][[3, 50]] = 0; rows["body"][[7, 90]] = B; rows["body"][20] = 0xfffffff0
        rows["position"][11, 1] = np.nan; rows["rotation"][12, 0] = np.inf
        rows["velocity"][13, 2] = np.nan; rows["angular_velocity"][14, 0] = -np.inf
        ok = valid(rows, fields, B)
        t_rows = torch.from_numpy(rows.view(np.int32).reshape(-1).copy()).cuda()
        t_skip = torch.full((1,), 12345, dtype=torch.int32, device="cuda")
        torch.cuda.synchronize()
        dev.set_body_states(None, fields, device_ptrs=(t_rows.data_ptr(), t_skip.data_ptr()), n=len(rows))
        torch.cuda.synchronize()
        assert int(t_skip.item()) == int((~ok).sum()) == {POSE: 7, VEL: 7, POSE | VEL: 9}[fields]
        with pytest.raises(nudge_b200.NudgeError):
            twin.set_body_states(rows, fields)   # the host path refuses the same list
        assert twin.set_body_states(rows[ok], fields) == 0
        assert _saved(dev) == _saved(twin), fields
        dev.step(); twin.step()
        assert _saved(dev) == _saved(twin), fields
    # all valid: skipped is written as 0, not accumulated; n = 0 writes 0 too
    rows = _random_rows(np.random.default_rng(3), B, 10)
    t_rows = torch.from_numpy(rows.view(np.int32).reshape(-1).copy()).cuda()
    for n in (10, 0):
        t_skip = torch.full((1,), 12345, dtype=torch.int32, device="cuda")
        torch.cuda.synchronize()
        dev.set_body_states(None, VEL, device_ptrs=(t_rows.data_ptr(), t_skip.data_ptr()), n=n)
        torch.cuda.synchronize()
        assert int(t_skip.item()) == 0, n


def _reset_loop(sim, ts, t_idx, t_out, t_skip, n):
    """get -> a torch op on the gathered rows (pull the position towards y = 3, halve the velocities) -> set, all on `ts`, the Sim's stream."""
    with torch.cuda.stream(ts):
        sim.get_body_states(device_ptrs=(t_idx.data_ptr(), t_out.data_ptr()), n=n)
        f = t_out.view(torch.float32).view(n, 16)
        f[:, 1] = f[:, 1] * 0.5 + 1.5
        f[:, 8:11] = f[:, 8:11] * 0.5
        f[:, 12:15] = f[:, 12:15] * 0.5
        sim.set_body_states(None, POSE | VEL, device_ptrs=(t_out.data_ptr(), t_skip.data_ptr()), n=n)


def test_a_captured_get_torch_op_set_graph_equals_the_same_calls_uncaptured():
    s = _scene(46)
    ts_a, ts_b = torch.cuda.Stream(), torch.cuda.Stream()
    a, b = _sim(s, ts_a.cuda_stream), _sim(s, ts_b.cuda_stream)
    n = 64
    idx = np.random.default_rng(4).choice(np.arange(8, s.n_bodies), n, replace=False).astype(np.uint32)
    bufs = {}
    for x, ts in ((a, ts_a), (b, ts_b)):
        with torch.cuda.stream(ts):
            for _ in range(10):
                x.step()
            bufs[x] = (torch.from_numpy(idx.view(np.int32)).cuda(), torch.zeros(n * 16, dtype=torch.int32, device="cuda"),
                       torch.zeros(1, dtype=torch.int32, device="cuda"))
    torch.cuda.synchronize()
    _reset_loop(a, ts_a, *bufs[a], n); _reset_loop(b, ts_b, *bufs[b], n)   # the first call allocates the set's scratch
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=ts_a):
        _reset_loop(a, ts_a, *bufs[a], n)
    torch.cuda.synchronize()
    records = a.debug_scalar("graph_records")
    for i in range(50):
        with torch.cuda.stream(ts_a):
            graph.replay()
        a.step()
        with torch.cuda.stream(ts_b):
            _reset_loop(b, ts_b, *bufs[b], n)
        b.step()
        if i % 10 == 9:
            torch.cuda.synchronize()
            assert _saved(a) == _saved(b), i
    torch.cuda.synchronize()
    assert _saved(a) == _saved(b)
    assert a.debug_scalar("graph_records") == records and a.debug_scalar("graph_active") == 1


def test_a_set_every_step_keeps_the_step_graph_and_its_launches():
    s = _scene(47)
    g = _sim(s)
    g.step(); g.step()
    records = g.debug_scalar("graph_records")
    ref = g.launch_count(); g.step(); per_step = g.launch_count() - ref
    rng = np.random.default_rng(6)
    for i in range(100):
        rows = _random_rows(rng, s.n_bodies, 8)
        fields = (POSE, VEL, POSE | VEL)[i % 3]
        c0 = g.launch_count()
        g.set_body_states(rows, fields)
        c1 = g.launch_count()
        assert c1 - c0 == (6 if fields & POSE else 3), i
        g.get_body_states(rows["body"])
        c2 = g.launch_count()
        assert c2 - c1 == 1
        g.step()
        assert g.launch_count() - c2 == per_step, i
    assert g.debug_scalar("graph_records") == records and g.debug_scalar("graph_active") == 1


def test_a_snapshot_before_a_reset_repeats_the_run_byte_for_byte():
    s = _scene(48)
    g = _sim(s)
    for _ in range(10):
        g.step()
    rows = _random_rows(np.random.default_rng(9), s.n_bodies, 50, kinematic=[7])
    snap = g.snapshot()
    run = []
    for i in range(20):
        if i == 4:
            g.set_body_states(rows, POSE | VEL)
        g.step()
        run.append(_saved(g))
    g.restore(snap)
    for i in range(20):
        if i == 4:
            g.set_body_states(rows, POSE | VEL)
        g.step()
        assert _saved(g) == run[i], i


def test_refusals_change_nothing():
    s = _scene(49)
    g = _sim(s)
    g.step_staged()
    before = _saved(g)
    L, ctx, st = g.lib, g.ctx, g.stream
    B = s.n_bodies
    good = _random_rows(np.random.default_rng(2), B, 6)
    P = lambda a: a.ctypes.data_as(ctypes.c_void_p)
    skip = ctypes.c_uint32(77)
    for fields in (0, 4, POSE | 8):
        assert L.nb_set_body_states(ctx, P(good), len(good), fields, ctypes.byref(skip), 0, st) == NB_ERR_ARGUMENT, fields
    for field, val, fields in (("body", 0, VEL), ("body", B, POSE), ("position", np.nan, POSE), ("rotation", np.inf, POSE | VEL),
                               ("velocity", np.nan, VEL), ("angular_velocity", -np.inf, POSE | VEL)):
        bad = good.copy()
        if field == "body":
            bad["body"][3] = val
        else:
            bad[field][3, 1] = val
        assert L.nb_set_body_states(ctx, P(bad), len(bad), fields, ctypes.byref(skip), 0, st) == NB_ERR_ARGUMENT, field
    assert L.nb_set_body_states(ctx, None, 3, VEL, None, 0, st) == NB_ERR_ARGUMENT
    assert L.nb_set_body_states(ctx, None, 3, VEL, None, 1, st) == NB_ERR_ARGUMENT
    idx = np.array([1, B], np.uint32)
    out = np.zeros(2, abi.BODY_STATE)
    assert L.nb_get_body_states(ctx, P(idx), 2, P(out), 0, st) == NB_ERR_ARGUMENT
    out = np.zeros(B + 1, abi.BODY_STATE)
    assert L.nb_get_body_states(ctx, None, B + 1, P(out), 0, st) == NB_ERR_ARGUMENT
    assert L.nb_get_body_states(ctx, P(idx), 2, None, 0, st) == NB_ERR_ARGUMENT
    assert _saved(g) == before
    # a NaN in a field the call does not select is not checked
    odd = good.copy(); odd["velocity"][2, 0] = np.nan
    assert g.set_body_states(odd, POSE) == 0
    # NB_BODY_POSE between nb_collide and nb_advance is refused; NB_BODY_VELOCITY alone is accepted there
    g.collide()
    mid = g.get_body_states().tobytes()
    for fields in (POSE, POSE | VEL):
        assert L.nb_set_body_states(ctx, P(good), len(good), fields, None, 0, st) == NB_ERR_ARGUMENT
    assert g.get_body_states().tobytes() == mid
    assert g.set_body_states(good, VEL) == 0
    g.apply_gravity_damping(); g.read_cached_impulses(); g.setup_contact_constraints(); g.apply_impulses(4)
    g.update_cached_impulses(); g.write_cached_impulses(); g.advance()
    assert g.set_body_states(good, POSE) == 0
    # a sharded context refuses a set (nothing changes); the gather still reads
    h = nudge_b200.Sim(s)
    h.step()
    h.shard_create(0, 1, None, 1, 1)
    before = h.get_body_states()
    with pytest.raises(nudge_b200.NudgeError, match="nb_shard_create"):
        h.set_body_states(good, VEL)
    assert h.get_body_states().tobytes() == before.tobytes()


def test_a_pose_set_refuses_a_connection_beyond_the_body_count():
    """nb_upload_connections accepts any body index; the wake needs both ends below B, so a pose set refuses such a set in both modes
    (nothing changes), as nb_remove_bodies does, while a velocity set, which wakes no partner, goes on and equals the restatement."""
    s = scenes.demo_scene(60, 60, iterations=4, spread=4.0, height=6.0, seed=50)
    B = s.n_bodies
    s.connections = np.array([(5, 6), (8, B + 3), (0xffffffff, 9)], scenes.PAIR32)
    g = nudge_b200.Sim(s, stream=side_stream())
    rows = _random_rows(np.random.default_rng(11), B, 20)
    before = g.get_body_states().tobytes()
    L, ctx, st = g.lib, g.ctx, g.stream
    t_rows = torch.from_numpy(rows.view(np.int32).reshape(-1).copy()).cuda()
    t_skip = torch.full((1,), 12345, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    for fields in (POSE, POSE | VEL):
        r = np.ascontiguousarray(rows)
        assert L.nb_set_body_states(ctx, r.ctypes.data_as(ctypes.c_void_p), len(r), fields, None, 0, st) == NB_ERR_ARGUMENT, fields
        assert L.nb_set_body_states(ctx, ctypes.c_void_p(t_rows.data_ptr()), len(r), fields, ctypes.c_void_p(t_skip.data_ptr()), 1, st) == NB_ERR_ARGUMENT, fields
        assert "connection 1" in L.nb_last_error(ctx).decode()
    torch.cuda.synchronize()
    assert g.get_body_states().tobytes() == before and int(t_skip.item()) == 12345
    # a velocity set is accepted, host and device mode, and writes what the restatement writes
    g.download_bodies()
    want, _ = set_states(live_scene(g), rows, VEL)
    assert g.set_body_states(rows, VEL) == 0
    g.download_bodies()
    assert (g.transforms.tobytes(), g.momentum.tobytes(), g.idle.tobytes()) == (want.transforms.tobytes(), want.momentum.tobytes(), want.idle.tobytes())
    g.set_body_states(None, VEL, device_ptrs=(t_rows.data_ptr(), t_skip.data_ptr()), n=len(rows))
    torch.cuda.synchronize()
    g.download_bodies()
    assert g.momentum.tobytes() == want.momentum.tobytes() and int(t_skip.item()) == 0
    # with the connections in range again a pose set runs, and wakes across them as the restatement does
    s.connections = np.array([(5, 6), (8, B - 3)], scenes.PAIR32)
    g.scene = s
    abi.HostState.__init__(g, s, g.cap)
    g.download_bodies()
    g._ck(L.nb_upload_connections(ctx, ctypes.byref(g.conn), st), "nb_upload_connections")
    g.idle[1:] = 0xff
    g.upload_bodies()
    moved = np.zeros(2, abi.BODY_STATE)
    moved["body"] = (8, 5); moved["rotation"][:, 3] = 1.0; moved["position"] = ((0.0, 20.0, 0.0), (3.0, 20.0, 0.0))
    g.download_bodies(); g.download_cache()
    want, woken = set_states(live_scene(g), moved, POSE, g.cache_view()["tags"])
    assert woken[B - 3] and woken[6]
    assert g.set_body_states(moved, POSE) == 0
    g.download_bodies()
    assert (g.transforms.tobytes(), g.momentum.tobytes(), g.idle.tobytes()) == (want.transforms.tobytes(), want.momentum.tobytes(), want.idle.tobytes())
