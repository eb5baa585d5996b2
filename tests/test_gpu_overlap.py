"""Overlap queries (nb_overlap; DESIGN.md section 8.15): offsets and hits byte for byte against the numpy brute force (oracle/overlap_ref.py)
on a settled 8k-box pile, a mixed box / sphere scene and the settled 65,536-box c2 pile, for small spheres around body centres, random
oriented boxes, points, large queries that test every collider, queries far outside the scene, queries touching colliders exactly and
degenerate queries; masks, sensors, ignore_body, kinematic bodies and body 0; after spawning, despawning and a snapshot restore.  Also: that
in-scene small queries walk the grid (also among sub-metre spheres on the standard ground), overflow, step invariance of a twin that
queries between every call, capture into a CUDA graph, buffers at 4-byte alignment, the launch count against torch.profiler and the
refusals."""
import json
import os
import subprocess
import sys
import numpy as np
import pytest
import torch
import nudge_b200
from nudge_b200 import abi, scenes
from oracle import overlap_ref, raycast_ref
from tests.gpu_util import side_stream
from tests.test_gpu_launch_count import LIBRARY_KERNEL
from tests.test_gpu_raycast import families as ray_families, small_mixed_scene, _state, _state_plain

pytestmark = pytest.mark.gpu
NAN, INF = float("nan"), float("inf")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SMALL = ("spheres", "boxes", "points", "touching")


def _oracle(sim, queries, flags=0):
    sim.download_bodies()
    scene = raycast_ref.Scene.of_sim(sim, getattr(sim.scene, "collision_filters", None), getattr(sim.scene, "sensors", None))
    return overlap_ref.query(scene, queries, flags)


def _same(sim, queries, flags=0, min_hits=1):
    off, hits = sim.overlap(queries, flags)
    want_off, want_hits = _oracle(sim, queries, flags)
    assert off.tobytes() == want_off.tobytes(), np.nonzero(off != want_off)[0][:5]
    if hits.tobytes() != want_hits.tobytes():
        q = np.setxor1d(hits.view(np.uint32).reshape(-1, 4)[:, 0], want_hits.view(np.uint32).reshape(-1, 4)[:, 0])
        raise AssertionError((len(hits), len(want_hits), q[:5]))
    assert len(hits) >= min_hits
    return off, hits


def _queries(n, shape):
    q = np.zeros(n, abi.OVERLAP_QUERY)
    q["shape"] = shape; q["mask"] = 0xffffffff; q["ignore_body"] = abi.RAY_NO_HIT; q["rotation"][:, 3] = 1.0
    return q


def _unit_quats(rng, n):
    v = rng.normal(size=(n, 4))
    return (v / np.linalg.norm(v, axis=1, keepdims=True)).astype(np.float32)


def families(sim, rng, n=256):
    """The query families, each of n queries, from the current transforms (the ground is box 0 on body 0 in these scenes)."""
    sim.download_bodies()
    p = sim.transforms["position"][1:]
    lo, hi = p.min(axis=0) - 2.0, p.max(axis=0) + 2.0
    span = float(np.linalg.norm(hi - lo))
    centres = p[rng.integers(0, len(p), n)]
    out = {}
    q = _queries(n, abi.OVERLAP_SPHERE); q["center"] = centres + rng.normal(size=(n, 3)) * 0.3; q["radius"] = rng.uniform(0.2, 1.5, n)
    out["spheres"] = q
    q = _queries(n, abi.OVERLAP_BOX); q["center"] = p[rng.integers(0, len(p), n)] + rng.normal(size=(n, 3)) * 0.3
    q["rotation"] = _unit_quats(rng, n); q["half_extents"] = rng.uniform(0.1, 2.0, (n, 3))
    q["rotation"][::5] = (0.0, 0.0, 0.0, 1.0)
    out["boxes"] = q
    q = _queries(n, abi.OVERLAP_SPHERE); q["center"] = rng.uniform(lo, hi, (n, 3))
    q["center"][::2] = p[rng.integers(0, len(p), len(q[::2]))]
    out["points"] = q
    # touching: spheres and axis-aligned boxes resting on the ground's top face, and spheres at a sphere collider's surface along an axis
    gy = sim.box_transforms["position"][0, 1]
    top = np.float32(gy + sim.box_data["size"][0, 1])
    q = _queries(n, abi.OVERLAP_SPHERE)
    q["radius"] = np.float32(0.5)
    q["center"] = np.c_[rng.uniform(lo[0], hi[0], n), np.full(n, np.float32(top + np.float32(0.5))), rng.uniform(lo[2], hi[2], n)]
    q["shape"][1::2] = abi.OVERLAP_BOX; q["half_extents"][1::2] = 0.5
    if len(sim.sphere_tags):
        k = rng.integers(0, len(sim.sphere_tags), n // 4)
        sp = raycast_ref.world_transforms(sim.transforms, sim.box_transforms, sim.sphere_transforms)["position"][len(sim.box_tags) + k]
        r = sim.sphere_data["radius"][k]
        q["shape"][::4] = abi.OVERLAP_SPHERE; q["radius"][::4] = 0.25
        q["center"][::4] = sp + np.c_[r + np.float32(0.25), np.zeros(len(k)), np.zeros(len(k))].astype(np.float32)
    out["touching"] = q
    q = _queries(16, abi.OVERLAP_SPHERE); q["center"] = 0.5 * (lo + hi); q["radius"] = span
    q["shape"][1::2] = abi.OVERLAP_BOX; q["half_extents"][1::2] = span; q["rotation"][1::2] = _unit_quats(rng, 8)
    q["rotation"][3] = (0.0, 0.0, 0.0, 2.0)   # not of unit length: used as given
    out["large"] = q
    d = rng.normal(size=(n, 3)); d /= np.linalg.norm(d, axis=1, keepdims=True)
    q = _queries(n, abi.OVERLAP_SPHERE); q["center"] = 0.5 * (lo + hi) + d * np.where(np.arange(n) % 2 == 0, 1e4, 1e7)[:, None]
    q["radius"] = 3.0; q["shape"][1::2] = abi.OVERLAP_BOX; q["half_extents"][1::2] = 3.0; q["rotation"][1::2] = _unit_quats(rng, n // 2)
    out["far"] = q
    q = _queries(12, abi.OVERLAP_SPHERE); q["center"] = 0.5 * (lo + hi); q["radius"] = 2.0; q["half_extents"] = 2.0
    q["shape"][6:] = abi.OVERLAP_BOX
    q["shape"][0] = 7; q["center"][1, 0] = NAN; q["radius"][2] = INF; q["radius"][3] = -1.0; q["radius"][4] = NAN; q["center"][5, 2] = -INF
    q["rotation"][6] = 0.0; q["rotation"][7, 1] = NAN; q["half_extents"][8, 0] = -0.5; q["half_extents"][9, 2] = INF; q["center"][10, 1] = NAN
    q["rotation"][11] = (1e-30, 0.0, 0.0, 1e-30)
    out["degenerate"] = q
    return out


def _settled(scene, steps):
    sim = nudge_b200.Sim(scene, stream=side_stream())
    for _ in range(steps):
        sim.step()
    return sim


@pytest.fixture(scope="module")
def pile8k():
    return _settled(scenes.box_drop(8192, seed=4), 300)


@pytest.fixture(scope="module")
def mixed():
    return _settled(scenes.demo_scene(2000, 2000, iterations=8, spread=12.0, height=30.0, seed=6), 200)


@pytest.mark.parametrize("scene", ["pile8k", "mixed"])
def test_every_family_equals_the_brute_force(scene, request):
    sim = request.getfixturevalue(scene)
    rng = np.random.default_rng(21)
    for name, q in families(sim, rng).items():
        off, hits = _same(sim, q, min_hits=0)
        if name == "degenerate":
            assert len(hits) == 0
        elif name in ("spheres", "boxes", "large"):
            assert (np.diff(off) > 0).sum() >= len(q) // 2, name


def test_in_scene_small_queries_walk_the_grid_and_large_ones_do_not(mixed):
    rng = np.random.default_rng(22)
    fam = families(mixed, rng)
    before = mixed.debug_scalar("overlap_fallbacks")
    for name in SMALL + ("degenerate",):
        _same(mixed, fam[name], min_hits=0)
    assert mixed.debug_scalar("overlap_fallbacks") == before
    _same(mixed, fam["large"])
    assert mixed.debug_scalar("overlap_fallbacks") > before   # at least the query whose rotation is not of unit length


def test_small_colliders_among_spheres_walk_the_grid():
    sim = _settled(small_mixed_scene(), 150)
    fam = families(sim, np.random.default_rng(23))
    for name in SMALL:
        _same(sim, fam[name])
    assert sim.debug_scalar("ray_grid_level") <= 8   # the queries' shared build
    assert sim.debug_scalar("overlap_fallbacks") == 0
    _same(sim, fam["far"], min_hits=0)


def test_c2_pile():
    sim = _settled(scenes.box_drop(65536, seed=2), 400)
    rng = np.random.default_rng(2048)
    q = np.concatenate([f[:512] for k, f in families(sim, rng, 512).items() if k in ("spheres", "boxes", "points", "touching")])
    assert len(q) == 2048
    off, hits = _same(sim, q)
    assert (hits["body"] == 0).any() and (np.diff(off) > 0).sum() > len(q) // 2


def test_masks_sensors_ignore_body_kinematic_and_body0(mixed):
    s = mixed.scene
    rng = np.random.default_rng(25)
    k = s.n_colliders
    filt = np.zeros(k, scenes.FILTER); filt["category"] = 1 << rng.integers(0, 4, k); filt["mask"] = 0xffff
    mixed.upload_collision_filters(filt)
    sens = (rng.random(k) < 0.2).astype(np.uint8); sens[0] = 0
    mixed.upload_sensors(sens)
    kin = np.zeros(20, scenes.KINEMATIC); kin["body"] = rng.choice(np.arange(1, s.n_bodies), 20, replace=False); kin["velocity"][:, 0] = 0.5
    mixed.upload_kinematic_bodies(kin)
    own = mixed._own_scene(); own.collision_filters, own.sensors = filt, sens
    for _ in range(5):
        mixed.step()
    fam = families(mixed, rng, 200)
    q = np.concatenate([fam["spheres"], fam["boxes"], fam["touching"]])
    q["mask"] = rng.choice([0x1, 0x3, 0x8, 0xf, 0x10, 0xffffffff], len(q))
    mixed.download_bodies()
    q["ignore_body"][::3] = rng.integers(0, s.n_bodies, len(q[::3]))
    q["ignore_body"][1::7] = 0
    for flags in (0, abi.OVERLAP_SENSORS):
        off, hits = _same(mixed, q, flags)
        assert sens[hits["collider"]].any() == bool(flags)
    kq = _queries(len(kin), abi.OVERLAP_SPHERE); kq["center"] = mixed.transforms["position"][kin["body"]]; kq["radius"] = 0.1
    off, hits = _same(mixed, kq)
    assert np.isin(hits["body"], kin["body"]).any()
    mixed.upload_kinematic_bodies(None); mixed.upload_sensors(None); mixed.upload_collision_filters(None)
    own.collision_filters, own.sensors = None, None


def test_after_spawning_despawning_and_a_snapshot_restore():
    s = scenes.box_drop(2048, seed=9)
    sim = nudge_b200.Sim(s, stream=side_stream(), max_bodies=s.n_bodies + 64, max_boxes=s.n_boxes + 64)
    for _ in range(100):
        sim.step()
    rng = np.random.default_rng(26)
    snap = sim.snapshot()
    before = families(sim, rng, 128)["spheres"]
    want = sim.overlap(before)
    sim.add_bodies(scenes.fragment(rng.uniform(-5, 5, (40, 3)) + (0.0, 40.0, 0.0), "box", first_tag=1 << 20))
    for name, q in families(sim, rng, 128).items():
        _same(sim, q, min_hits=0)
    sim.remove_bodies(np.arange(2, 400, 3))
    for name, q in families(sim, rng, 128).items():
        _same(sim, q, min_hits=0)
    for _ in range(20):
        sim.step()
    sim.restore(snap)
    off, hits = _same(sim, before)
    assert off.tobytes() == want[0].tobytes() and hits.tobytes() == want[1].tobytes()


def test_overflow_reports_the_total(pile8k):
    q = families(pile8k, np.random.default_rng(27), 64)["spheres"]
    want_off, want_hits = _oracle(pile8k, q)
    total = int(want_off[-1])
    assert total > 1
    offsets = np.zeros(len(q) + 1, np.uint32); hits = np.zeros(total - 1, abi.OVERLAP_HIT)
    r = pile8k.lib.nb_overlap(pile8k.ctx, abi.ptr(q), len(q), abi.ptr(hits), total - 1, abi.ptr(offsets), 0, 0, pile8k.stream)
    assert r == -2 and offsets[-1] == total
    with pytest.raises(nudge_b200.NudgeError):
        pile8k.overlap(q, capacity=total - 1)
    d_q = torch.from_numpy(q.view(np.uint8).copy()).cuda()
    d_h = torch.zeros(total * 16, dtype=torch.uint8, device="cuda")
    d_o = torch.zeros(len(q) + 1, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    pile8k.overlap(None, capacity=total - 1, device_ptrs=(d_q.data_ptr(), d_h.data_ptr(), d_o.data_ptr()), n=len(q))
    torch.cuda.synchronize()
    assert int(d_o.cpu()[-1]) == total
    pile8k.overlap(None, capacity=total, device_ptrs=(d_q.data_ptr(), d_h.data_ptr(), d_o.data_ptr()), n=len(q))
    torch.cuda.synchronize()
    assert d_o.cpu().numpy().view(np.uint32).tobytes() == want_off.tobytes()
    assert d_h.cpu().numpy().tobytes() == want_hits.tobytes()
    off, hits = pile8k.overlap(q)   # no capacity: the binding retries once with the total
    assert off.tobytes() == want_off.tobytes() and hits.tobytes() == want_hits.tobytes()


def test_querying_changes_nothing_a_step_observes():
    s = scenes.box_drop(4096, seed=7)
    a, b = nudge_b200.Sim(s, stream=side_stream()), nudge_b200.Sim(s, stream=side_stream())
    rng = np.random.default_rng(1)
    q = np.concatenate(list(families(a, rng, 64).values()))
    rays = np.concatenate(list(ray_families(a, rng, 32).values()))
    for g in (a, b):
        g.enable_contact_events(1 << 16)
    for step in range(100):
        for g in (a, b):
            g.step()
        a.overlap(q); a.raycast(rays)
        if step % 10 == 9:
            assert _state(a) == _state(b), step
    assert a.debug_scalar("graph_records") == b.debug_scalar("graph_records") == 1
    stages = ("collide", "apply_gravity_damping", "read_cached_impulses", "setup_contact_constraints", "apply_impulses", "update_cached_impulses",
              "write_cached_impulses", "advance")
    for _ in range(3):
        for st in stages:
            for g in (a, b):
                getattr(g, st)()
            a.overlap(q); a.raycast(rays)
    assert _state(a) == _state(b)


def test_capture_into_a_cuda_graph_replays_on_the_moved_scene():
    st = torch.cuda.Stream()
    s = scenes.box_drop(4096, seed=8)
    sim = nudge_b200.Sim(s, stream=st.cuda_stream)
    rng = np.random.default_rng(28)
    q = np.concatenate([f for k, f in families(sim, rng, 256).items()])
    n, cap = len(q), 1 << 20   # room for every hit: the large queries find thousands each
    d_q = torch.from_numpy(q.view(np.uint8).copy()).cuda()
    d_h = torch.zeros(cap * 16, dtype=torch.uint8, device="cuda")
    d_o = torch.zeros(n + 1, dtype=torch.int32, device="cuda")
    ptrs = (d_q.data_ptr(), d_h.data_ptr(), d_o.data_ptr())
    torch.cuda.synchronize()   # the Sim's stream is not ordered after torch's
    sim.overlap(None, capacity=cap, device_ptrs=ptrs, n=n)   # the first call allocates
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=st):
        sim.overlap(None, capacity=cap, device_ptrs=ptrs, n=n)
    for _ in range(3):
        for _ in range(15):
            sim.step()
        with torch.cuda.stream(st):
            d_h.zero_(); d_o.zero_()
            g.replay()
        st.synchronize()
        off = d_o.cpu().numpy().view(np.uint32)
        hits = d_h.cpu().numpy().view(abi.OVERLAP_HIT)[:off[-1]]
        fresh = sim.overlap(q)
        want = _oracle(sim, q)
        assert off.tobytes() == fresh[0].tobytes() == want[0].tobytes()
        assert hits.tobytes() == fresh[1].tobytes() == want[1].tobytes() and len(hits) > n // 2


def test_buffers_may_sit_at_any_4_byte_alignment(pile8k):
    q = families(pile8k, np.random.default_rng(29), 64)["boxes"]
    n, cap = len(q), 4096
    d_q = torch.zeros(n * 64 + 8, dtype=torch.uint8, device="cuda")
    d_q[4:4 + n * 64] = torch.from_numpy(q.view(np.uint8).copy()).cuda()
    hb = torch.full((cap * 16 + 16,), 0xab, dtype=torch.uint8, device="cuda")
    ob = torch.full(((n + 1) * 4 + 16,), 0xab, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    pile8k.overlap(None, capacity=cap, device_ptrs=(d_q.data_ptr() + 4, hb.data_ptr() + 4, ob.data_ptr() + 4), n=n)
    torch.cuda.synchronize()
    off, hits = pile8k.overlap(q)
    o = ob.cpu().numpy(); h = hb.cpu().numpy()
    assert o[4:4 + (n + 1) * 4].tobytes() == off.tobytes() and (o[:4] == 0xab).all() and (o[4 + (n + 1) * 4:] == 0xab).all()
    assert h[4:4 + len(hits) * 16].tobytes() == hits.tobytes() and (h[:4] == 0xab).all() and len(hits) > 0
    with pytest.raises(ValueError):
        pile8k.overlap(None, device_ptrs=(d_q.data_ptr(), hb.data_ptr(), ob.data_ptr()))


def _window(sim, calls, path):
    """Runs calls() under the profiler; returns (nb_launch_count delta, names of the kernel records)."""
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        torch.cuda.synchronize()
        before = sim.launch_count()
        calls()
        torch.cuda.synchronize()
        counted = sim.launch_count() - before
    prof.export_chrome_trace(str(path))
    with open(path) as f:
        names = [e["name"] for e in json.load(f)["traceEvents"] if e.get("ph") == "X" and e.get("cat") == "kernel"]
    return counted, names


def launch_count_windows(path):
    """The launch-count windows (host-pointer calls, device-pointer calls, calls between two graph-replayed steps): prints one JSON list of
    [expected, counted, kernel record names] per window.  Run in a process of its own by test_launch_count."""
    s = scenes.box_drop(2048, seed=3)
    sim = nudge_b200.Sim(s, stream=side_stream())
    sim.step()
    q = families(sim, np.random.default_rng(0), 64)["spheres"]
    n, cap = len(q), 4096
    d_q = torch.from_numpy(q.view(np.uint8).copy()).cuda()
    d_h = torch.zeros(cap * 16, dtype=torch.uint8, device="cuda")
    d_o = torch.zeros(n + 1, dtype=torch.int32, device="cuda")
    dev = lambda k=n: sim.overlap(None, capacity=cap, device_ptrs=(d_q.data_ptr(), d_h.data_ptr(), d_o.data_ptr()), n=k)
    torch.cuda.synchronize()   # the Sim's stream is not ordered after torch's
    sim.overlap(q, capacity=cap); dev()
    out = []
    for calls, want in ((lambda: (sim.overlap(q, capacity=cap), sim.overlap(q[:1], capacity=cap)), 18), (lambda: (dev(), dev(1)), 18),
                        (lambda: (sim.step(), sim.overlap(q, capacity=cap), dev(1), sim.step()), 2 * 61 + 18)):
        counted, names = _window(sim, calls, path)
        out.append([want, counted, names])
    print(json.dumps(out))


def test_launch_count(tmp_path):
    """nb_launch_count equals the header's 9 per call (1 without colliders) and the kernel records of torch.profiler, in a fresh process as
    for the ray casts (tests/test_gpu_raycast.py); the driver's memset32 kernels of a replayed step graph are not launches."""
    s = scenes.box_drop(2048, seed=3)
    sim = nudge_b200.Sim(s, stream=side_stream())
    sim.step()
    q = families(sim, np.random.default_rng(0), 64)["spheres"]
    sim.overlap(q, capacity=4096)
    before = sim.launch_count()
    sim.overlap(q, capacity=4096); sim.overlap(q[:1], capacity=4096)
    assert sim.launch_count() - before == 18
    off, hits = sim.overlap(q[:0])
    assert len(off) == 1 and off[0] == 0 and len(hits) == 0 and sim.launch_count() == before + 18   # n = 0: no launch
    code = "import tests.test_gpu_overlap as t; t.launch_count_windows(%r)" % str(tmp_path / "trace.json")
    r = subprocess.run([sys.executable] + (["-s"] if sys.flags.no_user_site else []) + ["-c", code], cwd=ROOT, capture_output=True, text=True,
                       timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    for want, counted, names in json.loads(r.stdout.strip().splitlines()[-1]):
        kernels = [k for k in names if k != "memset32"]
        assert [k for k in kernels if not LIBRARY_KERNEL.match(k)] == []
        assert len(kernels) == counted == want, sorted(set(kernels))
        assert sum(k.startswith("k_overlap(") or k == "k_overlap" for k in kernels) == 2
        assert sum(k.startswith("k_overlap_write") for k in kernels) == 2


def test_refusals_change_nothing():
    s = scenes.box_drop(512, seed=1)
    sim = nudge_b200.Sim(s)
    sim.step()
    q = families(sim, np.random.default_rng(0), 16)["spheres"]
    hits = np.zeros(64, abi.OVERLAP_HIT); off = np.zeros(len(q) + 1, np.uint32)
    want = _state_plain(sim)
    before = sim.launch_count()
    lib, P = sim.lib, abi.ptr
    assert lib.nb_overlap(sim.ctx, None, len(q), P(hits), 64, P(off), 0, 0, sim.stream) == -3
    assert lib.nb_overlap(sim.ctx, P(q), len(q), None, 64, P(off), 0, 0, sim.stream) == -3
    assert lib.nb_overlap(sim.ctx, P(q), len(q), P(hits), 64, None, 0, 0, sim.stream) == -3
    assert lib.nb_overlap(sim.ctx, P(q), len(q), P(hits), 64, P(off), 2, 0, sim.stream) == -3
    assert lib.nb_overlap(sim.ctx, None, 0, None, 0, None, 0, 1, sim.stream) == 0
    assert sim.launch_count() == before and hits.tobytes() == bytes(hits.nbytes) and off.tobytes() == bytes(off.nbytes)
    assert _state_plain(sim) == want
    sim.shard_create(0, 1, None, 16, 16)
    assert lib.nb_overlap(sim.ctx, P(q), len(q), P(hits), 64, P(off), 0, 0, sim.stream) == -3
    assert sim.launch_count() == before and hits.tobytes() == bytes(hits.nbytes) and off.tobytes() == bytes(off.nbytes)
    sim.close()
