"""Contact impulse reports on the device (nb_get_body_contact_impulses, nb_get_contact_pair_impulses; DESIGN.md section 8.22): bit identity
with tests/contact_impulse_ref.py fed nb_download_contacts, nb_debug_read("impulses") / ("sorted") and the transforms downloaded before the
step, on a pile and on demo_scene, in both solver modes, after nb_step and after the stage calls; host and device modes give the same bytes;
every NB_CONTACT_BEGIN event equals its pair row; the physics (momentum change, the weight on the ground, a resting box pushed up, a
kinematic platform's load); sleeping islands; the refusals; the calls that keep the report valid; no effect on the step or its launches;
and a captured step followed by both device calls."""
import ctypes as C
import os
import numpy as np
import pytest
import torch
import nudge_b200
from nudge_b200 import abi, scenes
from tests.contact_impulse_ref import REMOVED, body_report, pair_report
from tests.gpu_util import side_stream
from tests.kinematic_ref import with_kinematic_ground
from tests.test_body_impulse_oracle import settle_and_sleep, two_piles

pytestmark = pytest.mark.gpu
NB_ERR_ARGUMENT = -3


def _pile():
    return scenes.box_drop(1500, iterations=8, density_L=14.0, spacing=(2.2, 2.4, 2.2), rotate=True)


def _demo():
    return scenes.demo_scene(300, 300, iterations=8, spread=6.0, height=6.0, seed=11)


def _positions(g):
    g.download_bodies()
    return g.transforms["position"].copy()


def _inputs(g):
    g.download_contacts()
    cv = g.contacts_view()
    return cv["data"], cv["bodies"], cv["tags"], g.debug("impulses", scenes.IMPULSE), g.debug("sorted", np.uint32)


def _device_bodies(g, idx, n):
    out = torch.full((max(n, 1) * 8,), -1, dtype=torch.int32, device="cuda")
    t_idx = None if idx is None else torch.from_numpy(np.ascontiguousarray(idx, np.uint32).view(np.int32)).cuda()
    torch.cuda.synchronize()
    g.get_body_contact_impulses(device_ptrs=(None if t_idx is None else t_idx.data_ptr(), out.data_ptr()), n=n)
    torch.cuda.synchronize()
    return out.cpu().numpy().view(abi.BODY_CONTACT_IMPULSE)[:n]


def _device_pairs(g, thr, cap):
    out = torch.full((max(cap, 1) * 12,), -1, dtype=torch.int32, device="cuda")
    cnt = torch.full((1,), -1, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    g.get_contact_pair_impulses(thr, device_ptrs=(out.data_ptr(), cnt.data_ptr()), capacity=cap)
    torch.cuda.synchronize()
    c = int(cnt.item())
    return out.cpu().numpy().view(abi.CONTACT_PAIR_IMPULSE)[:min(c, cap)], c


def _check_against_restatement(g, pos):
    B = g.scene.n_bodies
    data, bodies, tags, imp, srt = _inputs(g)
    assert len(data) > 0
    want = body_report(data, bodies, imp, pos, B)
    got = g.get_body_contact_impulses()
    assert got.tobytes() == want.tobytes()
    rows, n = pair_report(data, bodies, tags, imp, srt)
    assert g.get_contact_pair_impulses().tobytes() == rows.tobytes()
    # device mode: the same bytes, also for a list with duplicates and indices past the body count
    assert _device_bodies(g, None, B).tobytes() == want.tobytes()
    idx = np.array([0, B - 1, 3, B, 3, REMOVED, 1], np.uint32)
    assert _device_bodies(g, idx, len(idx)).tobytes() == body_report(data, bodies, imp, pos, B, idx, device=True).tobytes()
    assert g.get_body_contact_impulses(idx[[0, 1, 2, 4, 6]]).tobytes() == want[idx[[0, 1, 2, 4, 6]]].tobytes()
    drows, dn = _device_pairs(g, -np.inf, n + 3)
    assert dn == n and drows.tobytes() == rows.tobytes()
    thr = float(np.median(rows["normal_impulse"]))
    kept, nk = pair_report(data, bodies, tags, imp, srt, thr)
    assert g.get_contact_pair_impulses(thr).tobytes() == kept.tobytes()
    part, pn = _device_pairs(g, thr, nk // 2)
    assert pn == nk and part.tobytes() == kept[:nk // 2].tobytes()
    return got, rows


@pytest.mark.parametrize("mode", ["parity", "throughput"])
@pytest.mark.parametrize("make", [_pile, _demo], ids=["pile", "demo"])
def test_reports_equal_the_restatement_after_nb_step_and_after_the_stage_calls(make, mode):
    s = make()
    g = nudge_b200.Sim(s, stream=side_stream())
    g.set_solver_mode(mode)
    for _ in range(60):
        g.step()
    for _ in range(2):
        pos = _positions(g)
        g.step()
        _check_against_restatement(g, pos)
    # the stage calls: the report is legal from the update on, and the write and the advance leave it unchanged
    pos = _positions(g)
    g.collide(); g.apply_gravity_damping(); g.read_cached_impulses(); g.setup_contact_constraints(); g.apply_impulses(int(s.iterations))
    g.update_cached_impulses()
    body, pairs = _check_against_restatement(g, pos)
    g.write_cached_impulses(); g.advance()
    assert g.get_body_contact_impulses().tobytes() == body.tobytes()
    assert g.get_contact_pair_impulses().tobytes() == pairs.tobytes()


def test_every_begin_event_equals_its_pair_row():
    g = nudge_b200.Sim(_demo(), stream=side_stream())
    g.enable_contact_events(1 << 16)
    begins = 0
    for _ in range(40):
        g.step()
        ev, dropped = g.contact_events()
        assert dropped == 0
        rows = g.get_contact_pair_impulses()
        by = {int(r["tags"]): r for r in rows}
        for e in ev[ev["kind"] == scenes.CONTACT_BEGIN]:
            r = by[int(e["tags"])]
            assert r["impulse"].tobytes() == e["impulse"].tobytes() and r["contacts"] == e["contacts"]
            assert r["penetration"].tobytes() == e["penetration"].tobytes() and (r["body_a"], r["body_b"]) == (e["body_a"], e["body_b"])
            begins += 1
    assert begins > 100


def _awake_settled(s, steps=150):
    """A Sim of s stepped through the stage calls until it rests, then every idle counter set to 0 (so the next step solves every island)."""
    g = nudge_b200.Sim(s)
    for _ in range(steps):
        g.step_staged()
    g.download_bodies()
    g.idle[:] = 0
    g.upload_bodies()
    return g


def test_body_impulse_is_the_momentum_change_and_the_ground_carries_the_weight():
    s, _, _ = two_piles(height=4)
    g = _awake_settled(s)
    g.collide(); g.apply_gravity_damping(); g.read_cached_impulses()
    g.download_bodies()
    v0 = g.momentum["velocity"].astype(np.float64)
    g.setup_contact_constraints(); g.apply_impulses(int(s.iterations))
    g.download_bodies()
    v1 = g.momentum["velocity"].copy()
    g.update_cached_impulses()
    rep = g.get_body_contact_impulses()
    minv = s.properties["mass_inverse"]
    dyn = np.nonzero(minv > 0)[0]
    assert len(dyn) == s.n_bodies - 1 and (rep["contacts"][dyn] > 0).all()
    m = (np.float64(1.0) / minv[dyn])[:, None]
    dp = m * (v1[dyn].astype(np.float64) - v0[dyn])
    got = rep["impulse"][dyn].astype(np.float64)
    # float32 velocities updated once per contact side and sweep: a few ulps of the velocity per update, in momentum units
    tol = 1e-4 * (np.abs(got) + m * np.abs(v0[dyn]) + m * 1e-3)
    assert (np.abs(dp - got) <= tol).all(), np.abs(dp - got).max()
    # at rest every dynamic body is pushed up by its own weight over the step, and the ground takes the whole weight: within 5 %
    w = np.float64(s.gravity) * np.float64(s.time_step)
    assert (got[:, 1] > 0).all()
    total = float((m[:, 0] * w).sum())
    assert abs(float(rep["impulse"][0][1]) + total) <= 0.05 * total
    assert abs(got[:, 1] - m[:, 0] * w).max() <= 0.25 * w * m.max()


def test_a_kinematic_platform_reports_the_load_it_carries_and_keeps_its_momentum():
    base, _, _ = two_piles(height=3)
    s, k = with_kinematic_ground(base)
    g = _awake_settled(s)
    before = g.momentum[k].copy()
    g.step_staged()
    g.download_bodies()
    assert g.momentum[k].tobytes() == before.tobytes()
    rep = g.get_body_contact_impulses(np.array([k, 0], np.uint32))
    minv = s.properties["mass_inverse"]
    dyn = [b for b in range(1, s.n_bodies) if b != k]
    total = float(sum(1.0 / minv[b] for b in dyn)) * float(s.gravity) * float(s.time_step)
    assert rep[0]["contacts"] > 0 and abs(float(rep[0]["impulse"][1]) + total) <= 0.05 * total
    assert rep[1]["contacts"] == 0 and (rep[1]["impulse"] == 0).all()   # body 0 carries no collider in this scene


def test_a_sleeping_island_reports_zeros_until_woken():
    s, pile_a, pile_b = two_piles()
    g = nudge_b200.Sim(s)
    settle_and_sleep(g)
    g.step_staged()
    rep = g.get_body_contact_impulses()
    assert (rep["contacts"] == 0).all() and (rep["impulse"] == 0).all() and (rep["angular_impulse"] == 0).all()
    st = g.get_body_states(pile_a)
    g.set_body_states(st, abi.BODY_VELOCITY)   # the same (zero) velocities: wakes exactly pile A
    g.step_staged()
    rep = g.get_body_contact_impulses()
    assert (rep["contacts"][pile_a] > 0).all() and (rep["contacts"][pile_b] == 0).all() and rep["contacts"][0] > 0
    assert (rep["impulse"][pile_b] == 0).all()


def _refused(g):
    """Both calls in both modes are NB_ERR_ARGUMENT and write nothing."""
    L, n = g.lib, g.scene.n_bodies
    hb = np.full(n * 32, 0x5A, np.uint8); hp = np.full(10 * 48, 0x5A, np.uint8); hc = np.full(1, 77, np.uint32)
    db = torch.full((n * 8,), 0x5A5A5A5A, dtype=torch.int32, device="cuda"); dp = torch.full((120,), 0x5A5A5A5A, dtype=torch.int32, device="cuda")
    dc = torch.full((1,), 77, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    assert L.nb_get_body_contact_impulses(g.ctx, None, n, abi.ptr(hb), 0, g.stream) == NB_ERR_ARGUMENT
    assert L.nb_get_body_contact_impulses(g.ctx, None, n, C.c_void_p(db.data_ptr()), 1, g.stream) == NB_ERR_ARGUMENT
    assert L.nb_get_contact_pair_impulses(g.ctx, -np.inf, abi.ptr(hp), 10, abi.ptr(hc), 0, g.stream) == NB_ERR_ARGUMENT
    assert L.nb_get_contact_pair_impulses(g.ctx, -np.inf, C.c_void_p(dp.data_ptr()), 10, C.c_void_p(dc.data_ptr()), 1, g.stream) == NB_ERR_ARGUMENT
    torch.cuda.synchronize()
    assert (hb == 0x5A).all() and (hp == 0x5A).all() and hc[0] == 77
    assert (db == 0x5A5A5A5A).all().item() and (dp == 0x5A5A5A5A).all().item() and dc.item() == 77


def _valid(g):
    return g.get_body_contact_impulses().tobytes() + g.get_contact_pair_impulses().tobytes()


def test_refusals_change_nothing(tmp_path):
    s = _demo()
    g = nudge_b200.Sim(s, stream=side_stream())
    _refused(g)   # a fresh context
    for _ in range(20):
        g.step()
    _valid(g)
    # the stage calls: refused from nb_collide until the update
    g.collide(); _refused(g)
    g.apply_gravity_damping(); _refused(g)
    g.read_cached_impulses(); _refused(g)
    g.setup_contact_constraints(); _refused(g)
    g.apply_impulses(4); _refused(g)
    g.update_cached_impulses(); _valid(g)
    g.write_cached_impulses(); g.advance(); _valid(g)
    snap = g.snapshot()
    path = str(tmp_path / "s.nbstate")
    g.save_state(path)
    L = g.lib

    def upload_contacts():
        g.download_contacts()
        g._ck(L.nb_upload_contacts(g.ctx, C.byref(g.contacts), None, g.stream), "nb_upload_contacts")

    def upload_bodies():
        g.download_bodies(); g.upload_bodies()

    clearing = {"nb_read_cached_impulses": g.read_cached_impulses, "nb_setup_contact_constraints": g.setup_contact_constraints,
                "nb_apply_impulses": lambda: g.apply_impulses(1), "nb_upload_contacts": upload_contacts, "nb_upload_bodies": upload_bodies,
                "nb_upload_colliders": lambda: g._ck(L.nb_upload_colliders(g.ctx, C.byref(g.colliders), g.stream), "nb_upload_colliders"),
                "nb_snapshot_restore": lambda: g.restore(snap), "nb_load_state": lambda: g.load_state(path),
                "nb_add_bodies": lambda: L.nb_add_bodies(g.ctx, None, None, None, g.stream),
                "nb_remove_bodies": lambda: g.remove_bodies([s.n_bodies - 1])}
    for name, call in clearing.items():
        g.step(); _valid(g)
        call()
        _refused(g)
    g.step()
    assert _valid(g)
    # a NaN threshold
    hc = np.full(1, 77, np.uint32)
    assert L.nb_get_contact_pair_impulses(g.ctx, float("nan"), None, 0, abi.ptr(hc), 0, g.stream) == NB_ERR_ARGUMENT and hc[0] == 77
    with pytest.raises(nudge_b200.NudgeError, match="NaN"):
        g.get_contact_pair_impulses(float("nan"))
    # host mode: an index past the body count, and a null list longer than the body count
    with pytest.raises(nudge_b200.NudgeError, match="body count"):
        g.get_body_contact_impulses([1, g.scene.n_bodies + 3])
    hb = np.zeros(g.scene.n_bodies + 1, abi.BODY_CONTACT_IMPULSE)
    assert L.nb_get_body_contact_impulses(g.ctx, None, len(hb), abi.ptr(hb), 0, g.stream) == NB_ERR_ARGUMENT
    # a sharded context
    h = nudge_b200.Sim(s)
    h.step()
    h.shard_create(0, 1, None, 1, 1)
    _refused(h)


def test_calls_that_keep_the_report_valid_leave_its_bytes():
    s = _demo()
    g = nudge_b200.Sim(s, stream=side_stream())
    for _ in range(25):
        g.step()
    want = _valid(g)
    g.apply_body_impulses([(5, (0.0, 0.0, 0.0), (0.0, 3.0, 0.0), (0.0, 0.0, 1.0), (0, 0))])
    st = g.get_body_states([3, 4, 9])
    st["velocity"] += 1.0
    g.set_body_states(st, abi.BODY_VELOCITY)
    rays = np.zeros(4, abi.RAY)
    rays["origin"] = (0.0, 20.0, 0.0); rays["direction"] = (0.0, -1.0, 0.0); rays["max_t"] = 100.0; rays["mask"] = 0xffff
    rays["ignore_body"] = 0xffffffff
    g.raycast(rays)
    g.get_body_states()
    assert _valid(g) == want


def _snapshot_outputs(x):
    x.download_bodies(); x.download_contacts(); x.download_cache()
    cv, kv = x.contacts_view(), x.cache_view()
    return (x.transforms.tobytes() + x.momentum.tobytes() + x.idle.tobytes() + b"".join(np.asarray(v).tobytes() for v in cv.values()) +
            b"".join(np.asarray(v).tobytes() for v in kv.values()))


def test_reports_change_nothing_the_step_computes_and_launch_what_the_header_says():
    s = _demo()
    a, b = nudge_b200.Sim(s, stream=side_stream()), nudge_b200.Sim(s, stream=side_stream())
    for x in (a, b):
        x.enable_contact_events(1 << 16)
    B = s.n_bodies
    idx = np.arange(0, B, 7, dtype=np.uint32)
    t_idx = torch.from_numpy(idx.view(np.int32)).cuda()
    ob = torch.zeros(B * 8, dtype=torch.int32, device="cuda"); op = torch.zeros(a.cap * 12, dtype=torch.int32, device="cuda")
    oc = torch.zeros(1, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()

    def launches(call):
        before = a.launch_count(); call(); return a.launch_count() - before

    for i in range(30):
        da, db = launches(a.step), b.launch_count()
        b.step()
        assert da == b.launch_count() - db
        if i >= 2:   # the scratch exists: host and device calls, their launches as the header states
            assert launches(lambda: a.get_body_contact_impulses(idx)) == 3
            assert launches(lambda: a.get_body_contact_impulses(device_ptrs=(t_idx.data_ptr(), ob.data_ptr()), n=len(idx))) == 3
            assert launches(lambda: a.get_body_contact_impulses(device_ptrs=(None, ob.data_ptr()), n=B)) == 3
            assert launches(lambda: a.get_contact_pair_impulses(0.0, capacity=a.cap)) == 5
            assert launches(lambda: a.get_contact_pair_impulses(device_ptrs=(op.data_ptr(), oc.data_ptr()), capacity=a.cap)) == 5
            assert launches(lambda: a.get_body_contact_impulses(np.zeros(0, np.uint32))) == 0
            assert launches(lambda: a.get_body_contact_impulses(device_ptrs=(None, ob.data_ptr()), n=0)) == 0
        else:
            a.get_body_contact_impulses(); a.get_contact_pair_impulses()
        if i % 10 == 9:
            ea, _ = a.contact_events(); eb, _ = b.contact_events()
            assert ea.tobytes() == eb.tobytes()
            assert _snapshot_outputs(a) == _snapshot_outputs(b)


def test_a_captured_step_and_both_reports_replay_the_uncaptured_bytes():
    s = _demo()
    B = s.n_bodies
    ts_a, ts_b = torch.cuda.Stream(), torch.cuda.Stream()
    old = os.environ.get("NB_GRAPH")
    os.environ["NB_GRAPH"] = "0"   # nb_step's own launches go into the application's graph
    try:
        a = nudge_b200.Sim(s, stream=ts_a.cuda_stream)
    finally:
        if old is None:
            del os.environ["NB_GRAPH"]
        else:
            os.environ["NB_GRAPH"] = old
    b = nudge_b200.Sim(s, stream=ts_b.cuda_stream)
    bufs = {}
    for x, ts in ((a, ts_a), (b, ts_b)):
        with torch.cuda.stream(ts):
            for _ in range(10):
                x.step()
            bufs[x] = (torch.zeros(B * 8, dtype=torch.int32, device="cuda"), torch.zeros(x.cap * 12, dtype=torch.int32, device="cuda"),
                       torch.zeros(1, dtype=torch.int32, device="cuda"))
    torch.cuda.synchronize()

    def step_and_report(x, ts):
        ob, op, oc = bufs[x]
        with torch.cuda.stream(ts):
            x.step()
            x.get_body_contact_impulses(device_ptrs=(None, ob.data_ptr()), n=B)
            x.get_contact_pair_impulses(device_ptrs=(op.data_ptr(), oc.data_ptr()), capacity=x.cap)

    step_and_report(a, ts_a); step_and_report(b, ts_b)   # the first calls allocate the scratch
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=ts_a):
        step_and_report(a, ts_a)
    torch.cuda.synchronize()
    for i in range(20):
        with torch.cuda.stream(ts_a):
            graph.replay()
        step_and_report(b, ts_b)
        torch.cuda.synchronize()
        (ab, ap, ac), (bb, bp, bc) = bufs[a], bufs[b]
        assert ac.item() == bc.item() > 0
        n = ac.item() * 12
        assert torch.equal(ab, bb) and torch.equal(ap[:n], bp[:n]), i
    assert _snapshot_outputs(a) == _snapshot_outputs(b)
