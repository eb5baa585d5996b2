"""Shape casts (nb_shapecast; DESIGN.md section 8.16): every hit byte for byte against the numpy brute force (oracle/shapecast_ref.py) on a
settled 8k-box pile, a mixed box / sphere scene, the settled 65,536-box c2 pile and a level-8 scene of sub-metre boxes and balls, for
spheres and boxes dropped onto the pile, sideways sweeps, random directions and rotations, casts starting inside or touching, casts
grazing the ground's face, long casts from far outside, large shapes and degenerate casts.  Also: sphere casts of radius 0 equal nb_raycast
and casts with max_t = 0 agree with nb_overlap, on the device; in-scene casts walk the grid while off-unit rotations and huge shapes fall
back; masks, sensors, ignore_body, kinematic bodies and body 0; after spawning, despawning and a snapshot restore; step invariance of a
twin that casts between every call; capture into a CUDA graph; buffers at 4-byte alignment; the launch count against torch.profiler; the
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
from oracle import raycast_ref, shapecast_ref
from tests.gpu_util import side_stream
from tests.test_gpu_launch_count import LIBRARY_KERNEL
from tests.test_gpu_raycast import families as ray_families, small_mixed_scene, _settled, _state, _state_plain, pile8k, mixed  # noqa: F401
from tests.test_gpu_overlap import families as overlap_families

pytestmark = pytest.mark.gpu
NAN, INF = float("nan"), float("inf")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
IN_SCENE = ("drop_spheres", "drop_boxes", "sideways", "random", "inside", "grazing", "degenerate")


def _oracle(sim, casts, flags=0):
    sim.download_bodies()
    scene = raycast_ref.Scene.of_sim(sim, getattr(sim.scene, "collision_filters", None), getattr(sim.scene, "sensors", None))
    return shapecast_ref.cast(scene, casts, flags)


def _same(sim, casts, flags=0, min_hits=1):
    got = sim.shapecast(casts, flags)
    want = _oracle(sim, casts, flags)
    bad = np.nonzero((got.view(np.uint8).reshape(-1, 48) != want.view(np.uint8).reshape(-1, 48)).any(axis=1))[0]
    assert not len(bad), (len(bad), casts[bad[:3]], got[bad[:3]], want[bad[:3]])
    assert (got["collider"] != abi.RAY_NO_HIT).sum() >= min_hits
    return got


def _casts(q, d, max_t):
    c = np.zeros(len(q), abi.SHAPE_CAST)
    c["shape"] = q; c["direction"] = d; c["max_t"] = max_t
    return c


def _dirs(rng, n):
    v = rng.normal(size=(n, 3))
    return v / np.linalg.norm(v, axis=1, keepdims=True)


def families(sim, rng, n=256):
    """The cast families, each of n casts (fewer for the large ones), from the current transforms; shapes from the overlap families."""
    ov = overlap_families(sim, rng, n)
    p = sim.transforms["position"][1:]
    lo, hi = p.min(axis=0) - 2.0, p.max(axis=0) + 2.0
    span = float(np.linalg.norm(hi - lo))
    mixed_shapes = np.concatenate([ov["spheres"][:n // 2], ov["boxes"][:n - n // 2]])
    out = {}
    for name, q in (("drop_spheres", ov["spheres"]), ("drop_boxes", ov["boxes"])):
        q = q.copy(); q["center"][:, 1] = hi[1] + 5.0
        out[name] = _casts(q, (0.0, -1.0, 0.0), 1e3)
    d = _dirs(rng, n); d[:, 1] = 0.0; d /= np.linalg.norm(d, axis=1, keepdims=True)
    out["sideways"] = _casts(mixed_shapes, d * rng.uniform(0.5, 2.0, (n, 1)), 20.0)
    q = mixed_shapes.copy(); q["center"] = rng.uniform(lo, hi, (n, 3))
    out["random"] = _casts(q, _dirs(rng, n) * rng.uniform(0.1, 3.0, (n, 1)), span)
    out["inside"] = _casts(ov["touching"], _dirs(rng, n), 5.0)
    t = ov["touching"].copy()   # resting exactly on the ground's top face, moving parallel to it
    out["grazing"] = _casts(t, np.where((np.arange(n) % 3 == 0)[:, None], (1.0, 0.0, 0.0), (1.0, 0.0, 0.25)), 1e3)
    out["grazing"]["shape"]["center"][:, 0] = lo[0] - 20.0
    out["grazing"]["shape"]["center"][1::2, 1] += np.float32(1e-3)   # half of them just clear of the face
    f = ov["far"]
    out["far"] = _casts(f, 0.5 * (lo + hi) - f["center"] + rng.normal(size=(len(f), 3)), np.where(np.arange(len(f)) % 3 == 0, 3e38, 2.0))
    q = ov["large"].copy(); q["rotation"][3] = (0.0, 0.0, 0.0, 1.0)
    q["center"] = 0.5 * (lo + hi) + np.array([0.0, 3.0 * span, 0.0])
    out["large"] = _casts(q, (0.0, -1.0, 0.0), 6.0 * span)
    q = ov["boxes"][:16].copy(); q["rotation"] = (0.0, 0.0, 0.0, 1.5); q["center"][:, 1] = hi[1] + 5.0   # off unit length: used as given
    out["off_unit"] = _casts(q, (0.0, -1.0, 0.0), 1e3)
    q = ov["spheres"][:12].copy(); q["center"] = 0.5 * (lo + hi)
    c = _casts(q, (0.0, -1.0, 0.0), 10.0)
    c["shape"]["shape"][0] = 7; c["direction"][1] = (NAN, 0.0, 0.0); c["direction"][2] = 0.0; c["direction"][3] = (-0.0, 0.0, -0.0)
    c["max_t"][4] = -1.0; c["max_t"][5] = NAN; c["max_t"][6] = INF; c["direction"][7, 2] = INF; c["shape"]["radius"][8] = -1.0
    c["shape"]["center"][9, 0] = NAN; c["shape"]["shape"][10] = abi.OVERLAP_BOX; c["shape"]["rotation"][10] = 0.0
    c["shape"]["shape"][11] = abi.OVERLAP_BOX; c["shape"]["half_extents"][11] = (1.0, -1.0, 1.0)
    out["degenerate"] = c
    return out


@pytest.mark.parametrize("scene", ["pile8k", "mixed"])
def test_every_family_equals_the_brute_force(scene, request):
    sim = request.getfixturevalue(scene)
    rng = np.random.default_rng(31)
    for name, c in families(sim, rng).items():
        got = _same(sim, c, min_hits=0)
        hits = (got["collider"] != abi.RAY_NO_HIT).sum()
        if name == "degenerate":
            assert hits == 0
        elif name in ("drop_spheres", "drop_boxes", "inside", "grazing", "large"):
            assert hits >= len(c) // 2, name
        if name == "inside":
            assert ((got["t"] == 0) & (got["collider"] != abi.RAY_NO_HIT)).sum() >= len(c) // 2


def test_in_scene_casts_walk_the_grid_and_huge_or_off_unit_ones_fall_back(mixed):
    fam = families(mixed, np.random.default_rng(32))
    before = mixed.debug_scalar("shapecast_fallbacks")
    for name in IN_SCENE:
        _same(mixed, fam[name], min_hits=0)
    assert mixed.debug_scalar("shapecast_fallbacks") == before
    _same(mixed, fam["off_unit"])
    assert mixed.debug_scalar("shapecast_fallbacks") == before + len(fam["off_unit"])
    _same(mixed, fam["large"])
    assert mixed.debug_scalar("shapecast_fallbacks") >= before + len(fam["off_unit"]) + len(fam["large"])


def test_level_8_scene_of_small_boxes_and_balls():
    sim = _settled(small_mixed_scene(), 150)
    fam = families(sim, np.random.default_rng(33))
    for name in IN_SCENE:
        _same(sim, fam[name], min_hits=0 if name in ("degenerate", "random") else 1)
    assert sim.debug_scalar("ray_grid_level") <= 8
    assert sim.debug_scalar("shapecast_fallbacks") == 0
    _same(sim, fam["far"], min_hits=0)


def test_c2_pile():
    sim = _settled(scenes.box_drop(65536, seed=2), 400)
    rng = np.random.default_rng(2048)
    fam = families(sim, rng, 512)
    c = np.concatenate([fam[k] for k in ("drop_spheres", "drop_boxes", "sideways", "inside")])
    assert len(c) == 2048
    got = _same(sim, c)
    assert (got["body"] == 0).any() and (got["collider"] != abi.RAY_NO_HIT).sum() > len(c) // 2


def _device_hits(sim, fn, n, buf):
    d_in = torch.from_numpy(buf.view(np.uint8).copy()).cuda()
    d_out = torch.zeros(n * 48, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    fn(None, device_ptrs=(d_in.data_ptr(), d_out.data_ptr()), n=n)
    torch.cuda.synchronize()
    return d_out.cpu().numpy().view(abi.RAY_HIT)


@pytest.mark.parametrize("scene", ["pile8k", "mixed"])
def test_radius_0_sphere_casts_equal_the_ray_casts(scene, request):
    sim = request.getfixturevalue(scene)
    rays = np.concatenate(list(ray_families(sim, np.random.default_rng(34)).values()))
    c = np.zeros(len(rays), abi.SHAPE_CAST)
    c["shape"]["shape"] = abi.OVERLAP_SPHERE; c["shape"]["center"] = rays["origin"]; c["shape"]["mask"] = rays["mask"]
    c["shape"]["ignore_body"] = rays["ignore_body"]; c["direction"] = rays["direction"]; c["max_t"] = rays["max_t"]
    want = _device_hits(sim, sim.raycast, len(rays), rays)
    got = _device_hits(sim, sim.shapecast, len(c), c)
    assert got.tobytes() == want.tobytes() and (got["collider"] != abi.RAY_NO_HIT).sum() > len(c) // 4


@pytest.mark.parametrize("scene", ["pile8k", "mixed"])
def test_max_t_0_casts_agree_with_the_overlap_queries(scene, request):
    sim = request.getfixturevalue(scene)
    rng = np.random.default_rng(35)
    ov = overlap_families(sim, rng)
    q = np.concatenate([ov[k] for k in ("spheres", "boxes", "points", "touching")])
    off, hits = sim.overlap(q)
    got = sim.shapecast(_casts(q, _dirs(rng, len(q)), 0.0))
    touching = 0
    for k in range(len(q)):
        mine = hits["collider"][off[k]:off[k + 1]]
        if len(mine):
            touching += 1
            assert got["t"][k] == 0.0 and got["collider"][k] <= mine.min(), k
    assert touching > len(q) // 4


def test_masks_sensors_ignore_body_kinematic_and_body0(mixed):
    s = mixed.scene
    rng = np.random.default_rng(36)
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
    c = np.concatenate([fam["drop_spheres"], fam["drop_boxes"], fam["sideways"], fam["inside"]])
    c["shape"]["mask"] = rng.choice([0x1, 0x3, 0x8, 0xf, 0x10, 0xffffffff], len(c))
    c["shape"]["ignore_body"][::3] = rng.integers(0, s.n_bodies, len(c[::3]))
    c["shape"]["ignore_body"][1::7] = 0
    for flags in (0, abi.SHAPECAST_SENSORS):
        got = _same(mixed, c, flags)
        hit = got["collider"][got["collider"] != abi.RAY_NO_HIT]
        assert sens[hit].any() == bool(flags)
    mixed.download_bodies()
    kc = _casts(overlap_families(mixed, rng, 20)["spheres"][:20], (0.0, -1.0, 0.0), 50.0)
    kc["shape"]["center"] = mixed.transforms["position"][kin["body"]] + (0.0, 3.0, 0.0); kc["shape"]["radius"] = 0.1
    got = _same(mixed, kc)
    assert np.isin(got["body"], kin["body"]).any()
    mixed.upload_kinematic_bodies(None); mixed.upload_sensors(None); mixed.upload_collision_filters(None)
    own.collision_filters, own.sensors = None, None


def test_after_spawning_despawning_and_a_snapshot_restore():
    s = scenes.box_drop(2048, seed=9)
    sim = nudge_b200.Sim(s, stream=side_stream(), max_bodies=s.n_bodies + 64, max_boxes=s.n_boxes + 64)
    for _ in range(100):
        sim.step()
    rng = np.random.default_rng(37)
    snap = sim.snapshot()
    before = families(sim, rng, 128)["drop_boxes"]
    want = sim.shapecast(before)
    sim.add_bodies(scenes.fragment(rng.uniform(-5, 5, (40, 3)) + (0.0, 40.0, 0.0), "box", first_tag=1 << 20))
    for name, c in families(sim, rng, 128).items():
        _same(sim, c, min_hits=0)
    sim.remove_bodies(np.arange(2, 400, 3))
    for name, c in families(sim, rng, 128).items():
        _same(sim, c, min_hits=0)
    for _ in range(20):
        sim.step()
    sim.restore(snap)
    got = _same(sim, before)
    assert got.tobytes() == want.tobytes()


def test_casting_changes_nothing_a_step_observes():
    s = scenes.box_drop(4096, seed=7)
    a, b = nudge_b200.Sim(s, stream=side_stream()), nudge_b200.Sim(s, stream=side_stream())
    rng = np.random.default_rng(1)
    c = np.concatenate([f[:64] for f in families(a, rng, 64).values()])
    for g in (a, b):
        g.enable_contact_events(1 << 16)
    for step in range(100):
        for g in (a, b):
            g.step()
        a.shapecast(c)
        if step % 10 == 9:
            assert _state(a) == _state(b), step
    assert a.debug_scalar("graph_records") == b.debug_scalar("graph_records") == 1
    stages = ("collide", "apply_gravity_damping", "read_cached_impulses", "setup_contact_constraints", "apply_impulses", "update_cached_impulses",
              "write_cached_impulses", "advance")
    for _ in range(3):
        for st in stages:
            for g in (a, b):
                getattr(g, st)()
            a.shapecast(c)
    assert _state(a) == _state(b)


def test_capture_into_a_cuda_graph_replays_on_the_moved_scene():
    st = torch.cuda.Stream()
    s = scenes.box_drop(4096, seed=8)
    sim = nudge_b200.Sim(s, stream=st.cuda_stream)
    rng = np.random.default_rng(38)
    c = np.concatenate([f for k, f in families(sim, rng, 128).items() if k != "large"])
    n = len(c)
    d_c = torch.from_numpy(c.view(np.uint8).copy()).cuda()
    d_h = torch.zeros(n * 48, dtype=torch.uint8, device="cuda")
    ptrs = (d_c.data_ptr(), d_h.data_ptr())
    torch.cuda.synchronize()   # the Sim's stream is not ordered after torch's
    sim.shapecast(None, device_ptrs=ptrs, n=n)   # the first call allocates
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=st):
        sim.shapecast(None, device_ptrs=ptrs, n=n)
    for _ in range(3):
        for _ in range(15):
            sim.step()
        with torch.cuda.stream(st):
            d_h.zero_()
            g.replay()
        st.synchronize()
        got = d_h.cpu().numpy().view(abi.RAY_HIT)
        fresh = sim.shapecast(c)
        assert got.tobytes() == fresh.tobytes() == _oracle(sim, c).tobytes()
        assert (got["collider"] != abi.RAY_NO_HIT).sum() > n // 4


def test_buffers_may_sit_at_any_4_byte_alignment(pile8k):
    c = families(pile8k, np.random.default_rng(39), 64)["drop_boxes"]
    n = len(c)
    d_c = torch.zeros(n * 80 + 8, dtype=torch.uint8, device="cuda")
    d_c[4:4 + n * 80] = torch.from_numpy(c.view(np.uint8).copy()).cuda()
    hb = torch.full((n * 48 + 16,), 0xab, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    pile8k.shapecast(None, device_ptrs=(d_c.data_ptr() + 4, hb.data_ptr() + 4), n=n)
    torch.cuda.synchronize()
    want = pile8k.shapecast(c)
    h = hb.cpu().numpy()
    assert h[4:4 + n * 48].tobytes() == want.tobytes() and (h[:4] == 0xab).all() and (h[4 + n * 48:] == 0xab).all()
    assert (want["collider"] != abi.RAY_NO_HIT).sum() > 0
    with pytest.raises(ValueError):
        pile8k.shapecast(None, device_ptrs=(d_c.data_ptr(), hb.data_ptr()))


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
    c = families(sim, np.random.default_rng(0), 64)["drop_spheres"]
    n = len(c)
    d_c = torch.from_numpy(c.view(np.uint8).copy()).cuda()
    d_h = torch.zeros(n * 48, dtype=torch.uint8, device="cuda")
    dev = lambda k=n: sim.shapecast(None, device_ptrs=(d_c.data_ptr(), d_h.data_ptr()), n=k)
    torch.cuda.synchronize()   # the Sim's stream is not ordered after torch's
    sim.shapecast(c); dev()
    out = []
    for calls, want in ((lambda: (sim.shapecast(c), sim.shapecast(c[:1])), 14), (lambda: (dev(), dev(1)), 14),
                        (lambda: (sim.step(), sim.shapecast(c), dev(1), sim.step()), 2 * 61 + 14)):
        counted, names = _window(sim, calls, path)
        out.append([want, counted, names])
    print(json.dumps(out))


def test_launch_count(tmp_path):
    """nb_launch_count equals the header's 7 per call (1 without colliders) and the kernel records of torch.profiler, in a fresh process as
    for the ray casts; the driver's memset32 kernels of a replayed step graph are not launches."""
    s = scenes.box_drop(2048, seed=3)
    sim = nudge_b200.Sim(s, stream=side_stream())
    sim.step()
    c = families(sim, np.random.default_rng(0), 64)["drop_spheres"]
    sim.shapecast(c)
    before = sim.launch_count()
    sim.shapecast(c); sim.shapecast(c[:1])
    assert sim.launch_count() - before == 14
    assert len(sim.shapecast(c[:0])) == 0 and sim.launch_count() == before + 14   # n = 0: no launch
    code = "import tests.test_gpu_shapecast as t; t.launch_count_windows(%r)" % str(tmp_path / "trace.json")
    r = subprocess.run([sys.executable] + (["-s"] if sys.flags.no_user_site else []) + ["-c", code], cwd=ROOT, capture_output=True, text=True,
                       timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    for want, counted, names in json.loads(r.stdout.strip().splitlines()[-1]):
        kernels = [k for k in names if k != "memset32"]
        assert [k for k in kernels if not LIBRARY_KERNEL.match(k)] == []
        assert len(kernels) == counted == want, sorted(set(kernels))
        assert sum(k.startswith("k_shapecast") for k in kernels) == 2


def test_refusals_change_nothing():
    s = scenes.box_drop(512, seed=1)
    sim = nudge_b200.Sim(s)
    sim.step()
    c = families(sim, np.random.default_rng(0), 16)["drop_spheres"]
    hits = np.zeros(len(c), abi.RAY_HIT)
    want = _state_plain(sim)
    before = sim.launch_count()
    lib, P = sim.lib, abi.ptr
    assert lib.nb_shapecast(sim.ctx, None, len(c), P(hits), 0, 0, sim.stream) == -3
    assert lib.nb_shapecast(sim.ctx, P(c), len(c), None, 0, 0, sim.stream) == -3
    assert lib.nb_shapecast(sim.ctx, P(c), len(c), P(hits), 2, 0, sim.stream) == -3
    assert lib.nb_shapecast(sim.ctx, None, 0, None, 0, 1, sim.stream) == 0
    assert sim.launch_count() == before and hits.tobytes() == bytes(hits.nbytes)
    assert _state_plain(sim) == want
    sim.shard_create(0, 1, None, 16, 16)
    assert lib.nb_shapecast(sim.ctx, P(c), len(c), P(hits), 0, 0, sim.stream) == -3
    assert sim.launch_count() == before and hits.tobytes() == bytes(hits.nbytes)
    sim.close()
