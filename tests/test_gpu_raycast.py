"""Ray casts (nb_raycast; DESIGN.md section 8.14): every hit byte for byte against the numpy brute force (oracle/raycast_ref.py) on a settled
8k-box pile, a mixed box / sphere scene and the settled 65,536-box c2 pile, for random rays, rays down onto the pile, rays from inside
colliders, rays parallel to the ground's faces, very long rays and rays from far outside, and degenerate rays; masks, sensors, ignore_body,
kinematic bodies and body 0; after spawning, despawning and a snapshot restore.  Also: the world transforms against nb_collide's, step
invariance of a twin that casts between every call, capture into a CUDA graph, the launch count against torch.profiler, the refusals, that
in-scene rays walk the grid (also among sub-metre spheres on the standard ground), and hit buffers at 4-byte alignment."""
import json
import os
import subprocess
import sys
import numpy as np
import pytest
import torch
import nudge_b200
from nudge_b200 import abi, scenes
from oracle import raycast_ref
from tests.gpu_util import side_stream
from tests.test_gpu_launch_count import LIBRARY_KERNEL

pytestmark = pytest.mark.gpu
NAN, INF = float("nan"), float("inf")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _oracle(sim, rays, flags=0):
    sim.download_bodies()
    scene = raycast_ref.Scene.of_sim(sim, getattr(sim.scene, "collision_filters", None), getattr(sim.scene, "sensors", None))
    return raycast_ref.cast(scene, rays, flags)


def _same(sim, rays, flags=0, min_hits=1):
    got = sim.raycast(rays, flags)
    want = _oracle(sim, rays, flags)
    bad = np.nonzero((got.view(np.uint8).reshape(-1, 48) != want.view(np.uint8).reshape(-1, 48)).any(axis=1))[0]
    assert not len(bad), (len(bad), rays[bad[:3]], got[bad[:3]], want[bad[:3]])
    assert (got["collider"] != abi.RAY_NO_HIT).sum() >= min_hits
    return got


def _rays(n):
    r = np.zeros(n, abi.RAY)
    r["mask"] = 0xffffffff; r["ignore_body"] = abi.RAY_NO_HIT
    return r


def _unit(rng, n):
    v = rng.normal(size=(n, 3))
    return v / np.linalg.norm(v, axis=1, keepdims=True)


def families(sim, rng, n=256):
    """The ray families, each of n rays, from the current transforms (the ground is collider 0 of these scenes)."""
    sim.download_bodies()
    p = sim.transforms["position"][1:]
    lo, hi = p.min(axis=0) - 2.0, p.max(axis=0) + 2.0
    span = float(np.linalg.norm(hi - lo))
    out = {}
    r = _rays(n); r["origin"] = rng.uniform(lo, hi, (n, 3)); r["direction"] = _unit(rng, n) * rng.uniform(0.1, 3.0, (n, 1)); r["max_t"] = span
    out["random"] = r
    r = _rays(n); r["origin"] = np.c_[rng.uniform(lo[0], hi[0], n), np.full(n, hi[1] + 5.0), rng.uniform(lo[2], hi[2], n)]
    r["direction"] = (0.0, -1.0, 0.0); r["max_t"] = 1e4
    out["down"] = r
    k = len(sim.box_tags) + len(sim.sphere_tags)
    pick = rng.integers(1, k, n)
    xf = np.concatenate([sim.box_transforms, sim.sphere_transforms])[pick]
    r = _rays(n); r["origin"] = sim.transforms["position"][xf["body"]] + rng.normal(size=(n, 3)) * 0.05; r["direction"] = _unit(rng, n); r["max_t"] = 50.0
    out["inside"] = r
    gy = sim.box_transforms["position"][0, 1]   # the ground: box 0 on body 0
    top = np.float32(gy + sim.box_data["size"][0, 1])
    r = _rays(n); r["origin"] = np.c_[rng.uniform(lo[0] - 20, lo[0], n), top + np.where(np.arange(n) % 2, 0.0, rng.uniform(0, 2, n)), rng.uniform(lo[2], hi[2], n)]
    r["direction"] = np.where((np.arange(n) % 3 == 0)[:, None], (1.0, 0.0, 0.0), (1.0, 0.0, 0.25)); r["max_t"] = 1e3
    r["origin"][::4, 1] = gy   # inside the ground, parallel to its faces
    out["parallel"] = r
    c = 0.5 * (lo + hi)
    dist = np.where(np.arange(n) % 2 == 0, 1e4, 1e7)[:, None]
    d = _unit(rng, n)
    r = _rays(n); r["origin"] = c + d * dist; r["direction"] = -d + rng.normal(size=(n, 3)) * 1e-3; r["max_t"] = np.where(np.arange(n) % 3 == 0, 3e38, 2e7)
    out["far"] = r
    r = _rays(8); r["origin"] = c; r["direction"] = (0.0, -1.0, 0.0); r["max_t"] = 10.0
    r["origin"][0, 0] = NAN; r["direction"][1, 2] = INF; r["direction"][2] = 0.0; r["max_t"][3] = -1.0; r["max_t"][4] = NAN; r["max_t"][5] = INF
    r["direction"][6] = (-0.0, 0.0, -0.0); r["origin"][7, 1] = -INF
    out["degenerate"] = r
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


def test_world_transforms_equal_the_collide(pile8k):
    pile8k.collide()
    got = pile8k.debug("world_xf", scenes.TRANSFORM)
    pile8k.download_bodies()
    want = raycast_ref.world_transforms(pile8k.transforms, pile8k.box_transforms, pile8k.sphere_transforms)
    assert got.tobytes() == want.tobytes()
    pile8k.step()   # end the step the collide began


@pytest.mark.parametrize("scene", ["pile8k", "mixed"])
def test_every_family_equals_the_brute_force(scene, request):
    sim = request.getfixturevalue(scene)
    rng = np.random.default_rng(11)
    for name, rays in families(sim, rng).items():
        got = _same(sim, rays, min_hits=0)
        hits = (got["collider"] != abi.RAY_NO_HIT).sum()
        if name == "degenerate":
            assert hits == 0
        elif name in ("down", "inside", "parallel"):
            assert hits >= len(rays) // 2, name


def _grid_fallbacks(sim):
    return sim.debug_scalar("ray_fallbacks")


def test_in_scene_rays_walk_the_grid(mixed):
    """Rays inside the scene never fall back to testing every collider, also among spheres; only origins far outside may."""
    rng = np.random.default_rng(12)
    fam = families(mixed, rng)
    before = _grid_fallbacks(mixed)
    for name in ("random", "down", "inside", "parallel", "degenerate"):
        _same(mixed, fam[name], min_hits=0)
    assert _grid_fallbacks(mixed) == before


def small_mixed_scene(n=3000, seed=13):
    """Sub-metre boxes and balls (half extents and radii 0.15 to 0.35) dropped on the standard 400-half-extent ground: every collider spans
    under 1/256 of the Morton frame's extent, so the grid level is 8 or finer."""
    rng = np.random.default_rng(seed)
    nb = n // 2
    sizes = (rng.random((nb, 3)) * 0.2 + 0.15).astype(np.float32)
    radii = (rng.random(n - nb) * 0.2 + 0.15).astype(np.float32)
    pos = lambda k: np.stack([rng.uniform(-8, 8, k), rng.uniform(0, 25, k) - 9.0, rng.uniform(-8, 8, k)], 1).astype(np.float32)
    return scenes._assemble("small_mixed", sizes, pos(nb), scenes._random_unit_quaternions(rng, nb), radii, pos(n - nb))


def test_small_colliders_among_spheres_walk_the_grid():
    sim = _settled(small_mixed_scene(), 150)
    rng = np.random.default_rng(14)
    fam = families(sim, rng)
    for name in ("random", "down", "inside", "parallel"):
        _same(sim, fam[name])
    assert sim.debug_scalar("ray_grid_level") <= 8
    assert _grid_fallbacks(sim) == 0
    _same(sim, fam["far"], min_hits=0)   # origins 10^4 and 10^7 away: these may test every collider, with the same result


def test_hits_may_be_written_at_any_4_byte_alignment(pile8k):
    """nb_ray and nb_ray_hit are 4-byte aligned structs: rays read from and hits written to buffers 4 bytes past a 16-byte boundary."""
    rays = families(pile8k, np.random.default_rng(15), 64)["random"]
    n = len(rays)
    d_rays = torch.zeros(n * 48 + 8, dtype=torch.uint8, device="cuda")
    d_rays[4:4 + n * 48] = torch.from_numpy(rays.view(np.uint8).copy()).cuda()
    buf = torch.full((n * 48 + 16,), 0xab, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()   # the Sim's stream is not ordered after torch's
    pile8k.raycast(None, device_ptrs=(d_rays.data_ptr() + 4, buf.data_ptr() + 4), n=n)
    torch.cuda.synchronize()
    out = buf.cpu().numpy()
    assert out[4:4 + n * 48].tobytes() == pile8k.raycast(rays).tobytes()
    assert (out[:4] == 0xab).all() and (out[4 + n * 48:] == 0xab).all()
    with pytest.raises(ValueError):
        pile8k.raycast(None, device_ptrs=(d_rays.data_ptr(), buf.data_ptr()))


def test_c2_pile():
    sim = _settled(scenes.box_drop(65536, seed=2), 400)
    rng = np.random.default_rng(2048)
    rays = np.concatenate([f[:512] for k, f in families(sim, rng, 512).items() if k != "degenerate"])
    assert len(rays) >= 2048
    got = _same(sim, rays)
    assert (got["body"] == 0).any() and (got["body"] > 0).sum() > len(rays) // 4


def test_masks_sensors_ignore_body_kinematic_and_body0(mixed):
    s = mixed.scene
    rng = np.random.default_rng(5)
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
    rays = np.concatenate([fam["random"], fam["down"], fam["inside"]])
    rays["mask"] = rng.choice([0x1, 0x3, 0x8, 0xf, 0x10, 0xffffffff], len(rays))
    mixed.download_bodies()
    rays["ignore_body"][::3] = rng.integers(0, s.n_bodies, len(rays[::3]))
    rays["ignore_body"][1::7] = 0
    for flags in (0, abi.RAY_SENSORS):
        got = _same(mixed, rays, flags)
        if flags:
            assert sens[got["collider"][got["collider"] != abi.RAY_NO_HIT]].any()
    down = fam["down"].copy()
    assert (mixed.raycast(down)["body"] == 0).any()
    kr = _rays(len(kin)); kr["origin"] = mixed.transforms["position"][kin["body"]] + (0.0, 30.0, 0.0); kr["direction"] = (0.0, -1.0, 0.0); kr["max_t"] = 100.0
    got = _same(mixed, kr)
    assert np.isin(got["body"], kin["body"]).any()
    mixed.upload_kinematic_bodies(None); mixed.upload_sensors(None); mixed.upload_collision_filters(None)
    own.collision_filters, own.sensors = None, None


def test_after_spawning_despawning_and_a_snapshot_restore():
    s = scenes.box_drop(2048, seed=9)
    sim = nudge_b200.Sim(s, stream=side_stream(), max_bodies=s.n_bodies + 64, max_boxes=s.n_boxes + 64)
    for _ in range(100):
        sim.step()
    rng = np.random.default_rng(3)
    snap = sim.snapshot()
    before = families(sim, rng, 128)
    want = sim.raycast(before["down"])
    sim.add_bodies(scenes.fragment(rng.uniform(-5, 5, (40, 3)) + (0.0, 40.0, 0.0), "box", first_tag=1 << 20))
    for name, rays in families(sim, rng, 128).items():
        _same(sim, rays, min_hits=0)
    sim.remove_bodies(np.arange(2, 400, 3))
    for name, rays in families(sim, rng, 128).items():
        _same(sim, rays, min_hits=0)
    for _ in range(20):
        sim.step()
    sim.restore(snap)
    got = _same(sim, before["down"])
    assert got.tobytes() == want.tobytes()


def _state(g):
    g.download_bodies(); g.download_cache()
    c = g.counts()
    ev, dropped = g.contact_events()
    return g.transforms.tobytes() + g.momentum.tobytes() + g.idle.tobytes() + g.cache_tags[:g.cache.count].tobytes() + \
        g.cache_data[:g.cache.count].tobytes() + bytes(c) + ev.tobytes() + bytes([dropped])


def test_casting_changes_nothing_a_step_observes():
    s = scenes.box_drop(4096, seed=7)
    a, b = nudge_b200.Sim(s, stream=side_stream()), nudge_b200.Sim(s, stream=side_stream())
    rng = np.random.default_rng(1)
    rays = np.concatenate(list(families(a, rng, 64).values()))
    for g in (a, b):
        g.enable_contact_events(1 << 16)
    for step in range(100):
        for g in (a, b):
            g.step()
        a.raycast(rays)
        if step % 10 == 9:
            assert _state(a) == _state(b), step
    assert a.debug_scalar("graph_records") == b.debug_scalar("graph_records") == 1
    stages = ("collide", "apply_gravity_damping", "read_cached_impulses", "setup_contact_constraints", "apply_impulses", "update_cached_impulses",
              "write_cached_impulses", "advance")
    for _ in range(3):
        for st in stages:
            for g in (a, b):
                getattr(g, st)()
            a.raycast(rays)
    assert _state(a) == _state(b)


def test_capture_into_a_cuda_graph_replays_on_the_moved_scene():
    st = torch.cuda.Stream()
    s = scenes.box_drop(4096, seed=8)
    sim = nudge_b200.Sim(s, stream=st.cuda_stream)
    rng = np.random.default_rng(4)
    rays = np.concatenate([f for k, f in families(sim, rng, 256).items()])
    n = len(rays)
    d_rays = torch.from_numpy(rays.view(np.uint8).copy()).cuda()
    d_hits = torch.zeros(n * 48, dtype=torch.uint8, device="cuda")
    ptrs = (d_rays.data_ptr(), d_hits.data_ptr())
    torch.cuda.synchronize()   # the Sim's stream is not ordered after torch's
    sim.raycast(None, device_ptrs=ptrs, n=n)   # the first call allocates
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=st):
        sim.raycast(None, device_ptrs=ptrs, n=n)
    for _ in range(3):
        for _ in range(15):
            sim.step()
        with torch.cuda.stream(st):
            d_hits.zero_()
            g.replay()
        st.synchronize()
        got = d_hits.cpu().numpy().view(abi.RAY_HIT)
        fresh = sim.raycast(rays)
        assert got.tobytes() == fresh.tobytes() == _oracle(sim, rays).tobytes()


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
    rays = families(sim, np.random.default_rng(0), 64)["random"]
    n = len(rays)
    d_rays = torch.from_numpy(rays.view(np.uint8).copy()).cuda()
    d_hits = torch.zeros(n * 48, dtype=torch.uint8, device="cuda")
    dev = lambda k=n: sim.raycast(None, device_ptrs=(d_rays.data_ptr(), d_hits.data_ptr()), n=k)
    torch.cuda.synchronize()   # the Sim's stream is not ordered after torch's
    sim.raycast(rays); dev()
    out = []
    for calls, want in ((lambda: (sim.raycast(rays), sim.raycast(rays[:1])), 14), (lambda: (dev(), dev(1)), 14),
                        (lambda: (sim.step(), sim.raycast(rays), dev(1), sim.step()), 2 * 61 + 14)):
        counted, names = _window(sim, calls, path)
        out.append([want, counted, names])
    print(json.dumps(out))


def test_launch_count(tmp_path):
    """nb_launch_count equals the header's 7 per call and the kernel records of torch.profiler.  A replayed step graph's memset nodes (the
    step's cudaMemsetAsync calls) appear in the trace as the driver's "memset32" kernels; they are not launches.  The windows run in a fresh
    process: late in a long GPU test session the profiler's trace of the same windows held only some of the kernel records (2 of 14) while
    the launch count and every result were right, and a fresh process gives the whole trace."""
    s = scenes.box_drop(2048, seed=3)
    sim = nudge_b200.Sim(s, stream=side_stream())
    sim.step()
    rays = families(sim, np.random.default_rng(0), 64)["random"]
    sim.raycast(rays)
    before = sim.launch_count()
    sim.raycast(rays); sim.raycast(rays[:1])
    assert sim.launch_count() - before == 14
    assert len(sim.raycast(rays[:0])) == 0 and sim.launch_count() == before + 14   # n = 0: no launch
    code = "import tests.test_gpu_raycast as t; t.launch_count_windows(%r)" % str(tmp_path / "trace.json")
    r = subprocess.run([sys.executable] + (["-s"] if sys.flags.no_user_site else []) + ["-c", code], cwd=ROOT, capture_output=True, text=True,
                       timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    for want, counted, names in json.loads(r.stdout.strip().splitlines()[-1]):
        kernels = [k for k in names if k != "memset32"]
        assert [k for k in kernels if not LIBRARY_KERNEL.match(k)] == []
        assert len(kernels) == counted == want, sorted(set(kernels))
        assert sum(k.startswith("k_raycast") for k in kernels) == 2


def test_refusals_change_nothing():
    s = scenes.box_drop(512, seed=1)
    sim = nudge_b200.Sim(s)
    sim.step()
    rays = families(sim, np.random.default_rng(0), 16)["random"]
    hits = np.zeros(len(rays), abi.RAY_HIT)
    want = _state_plain(sim)
    before = sim.launch_count()
    lib = sim.lib
    assert lib.nb_raycast(sim.ctx, None, len(rays), abi.ptr(hits), 0, 0, sim.stream) == -3
    assert lib.nb_raycast(sim.ctx, abi.ptr(rays), len(rays), None, 0, 0, sim.stream) == -3
    assert lib.nb_raycast(sim.ctx, abi.ptr(rays), len(rays), abi.ptr(hits), 2, 0, sim.stream) == -3
    assert lib.nb_raycast(sim.ctx, None, 0, None, 0, 1, sim.stream) == 0
    assert sim.launch_count() == before and hits.tobytes() == bytes(hits.nbytes) and _state_plain(sim) == want
    sim.shard_create(0, 1, None, 16, 16)
    assert lib.nb_raycast(sim.ctx, abi.ptr(rays), len(rays), abi.ptr(hits), 0, 0, sim.stream) == -3
    assert sim.launch_count() == before and hits.tobytes() == bytes(hits.nbytes)
    sim.close()


def _state_plain(g):
    g.download_bodies()
    return g.transforms.tobytes() + g.momentum.tobytes() + g.idle.tobytes()
