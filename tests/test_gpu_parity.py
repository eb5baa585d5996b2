"""GPU parity tests proper: the CUDA path through the C ABI against the CPU oracle on the same seeded inputs, bit for
bit at every stage (pair lists, contacts, tag order, batch indices, constraint rows, impulses after every sweep,
momentum, cache, transforms), against the committed golden fixtures, and through size-independent properties at the
full BASELINE size."""
import os
import numpy as np
import pytest
import nudge_b200
from nudge_b200 import scenes, abi
from tests import golden_util as G
from tests.parity_util import Report, compare_oracle_gpu_step, sync_oracle_from_gpu

pytestmark = pytest.mark.gpu


def _pair(scene):
    from oracle import pyoracle
    o = pyoracle.OracleSim(scene)
    g = nudge_b200.Sim(scene, contact_capacity=o.cap, debug=True)
    assert g.lut_model_exact(), "host CPU's rcpps/rsqrtps do not follow the LUT model: bit parity is not expected on this box"
    return o, g


def _steps(o, g, n, individually=True):
    for i in range(n):
        rep = Report("%s step %d" % (o.scene.name, i))
        assert compare_oracle_gpu_step(o, g, rep, individually), str(rep)
        assert g.counts().overflow == 0


def test_library_is_the_cuda_extension():
    g = nudge_b200.Sim(scenes.two_boxes())
    g.collide(); g.download_contacts()
    assert g.launch_count() > 10 and g.contacts.count == 8  # two unit boxes face to face: the 8-point manifold


def test_device_lut_equals_host_instruction():
    from oracle import pyoracle
    lib = pyoracle.load()
    g = nudge_b200.Sim(scenes.demo_scene(2000, 0))
    rng = np.random.default_rng(0)
    x = rng.integers(0, 2**32, 1 << 16, dtype=np.uint64).astype(np.uint32).view(np.float32)
    for rs in (False, True):
        y = np.empty_like(x); (lib.nbo_rsqrt if rs else lib.nbo_rcp)(abi.ptr(x), abi.ptr(y), len(x))
        yd = g.device_rcp(x, rs)
        same = (y.view(np.uint32) == yd.view(np.uint32)) | (np.isnan(y) & np.isnan(yd))
        assert same.all()


def test_small_mixed_scene_every_stage():
    o, g = _pair(scenes.demo_scene(100, 100, iterations=4, spread=2.0, height=20.0))
    _steps(o, g, 25)


def test_demo_scene_config0():
    o, g = _pair(scenes.demo_scene(1024, 1024, iterations=8))
    _steps(o, g, 10)


def test_rotated_box_drop():
    o, g = _pair(scenes.box_drop(3000, iterations=8))
    _steps(o, g, 30)


def test_fused_sweeps_equal_individual_sweeps():
    o, g = _pair(scenes.demo_scene(300, 300, iterations=16, spread=4.0, height=80.0))
    _steps(o, g, 6, individually=False)


def test_sleeping_islands_and_culled_cache():
    o, g = _pair(scenes.demo_scene(120, 120, iterations=4, spread=6.0, height=6.0, seed=11))
    _steps(o, g, 40)
    rng = np.random.default_rng(5)
    sleepy = rng.random(o.scene.n_bodies) < 0.8
    for s in (o, g):
        s.idle[sleepy] = 0xff
        s.momentum["velocity"][sleepy] = 0; s.momentum["angular_velocity"][sleepy] = 0
    g.upload_bodies()
    seen = 0
    for i in range(6):
        rep = Report("sleep %d" % i)
        assert compare_oracle_gpu_step(o, g, rep), str(rep)
        seen = max(seen, g.contacts.sleeping_count)
    assert seen > 0


def test_empty_and_contact_free_scenes():
    s = scenes.demo_scene(0, 0)               # ground only
    o, g = _pair(s); _steps(o, g, 2)
    s = scenes.demo_scene(20, 20, spread=50.0, height=300.0)   # nothing touches
    o, g = _pair(s); _steps(o, g, 3)


def test_golden_two_box_cases_through_cuda():
    """The reference's own known-answer tests (tests/main.cpp), run on the GPU path: counts 4 / 8 / 3 / 1 / 2 and exact tags."""
    g0 = G.load_box_cases()
    sim = nudge_b200.Sim(G.scene_of(g0, 0), contact_capacity=64)
    errs = []
    for k in range(len(g0["count"])):
        s = G.scene_of(g0, k)
        sim.transforms[:] = s.transforms; sim.box_data[:] = s.box_data; sim.box_transforms[:] = s.box_transforms
        sim.upload()
        sim.collide(); sim.download_contacts()
        e = G.check_case(g0, k, sim.contacts_view())
        if e:
            errs.append(e)
    assert not errs, "\n".join(errs[:10])


def test_golden_trajectory_through_cuda():
    t = np.load(os.path.join(G.HERE, "golden", "step_cases.npz"))
    s = scenes.demo_scene(48, 48, iterations=8, seed=int(t["seed"]), spread=2.0, height=12.0)
    g = nudge_b200.Sim(s)
    for k in range(len(t["contacts"])):
        g.step()
        g.download_bodies()
        c = g.counts()
        assert c.contacts == t["contacts"][k] and c.cache == t["cache"][k]
        assert np.array_equal(g.transforms.view(np.uint8), t["transforms"][k].view(np.uint8)), "transforms differ at step %d" % k
        assert np.array_equal(g.momentum.view(np.uint8), t["momentum"][k].view(np.uint8)), "momentum differs at step %d" % k


def test_settled_8k_pile_one_step_from_identical_state():
    s = scenes.box_drop(8000, iterations=8)
    o, g = _pair(s)
    for _ in range(500):
        g.step()
    sync_oracle_from_gpu(o, g)
    _steps(o, g, 2)


def test_full_size_64k_properties_and_one_step_parity():
    """BASELINE config 1 size: 65,536 boxes.  Settles on the GPU, then (a) one full step bit-exact against the widened
    oracle from identical state and (b) size-independent properties: pair list sorted and unique, every pair's AABBs
    overlap, contact tag order sorted, batches conflict-free."""
    s = scenes.box_drop(65536, iterations=8)
    o, g = _pair(s)
    for _ in range(700):
        g.step()
    assert g.counts().overflow == 0
    sync_oracle_from_gpu(o, g)
    _steps(o, g, 1)
    g.collide(); g.apply_gravity_damping(); g.read_cached_impulses(); g.setup_contact_constraints()
    g.download_contacts()
    p = g.pairs_view()
    key = (p["hi"].astype(np.uint64) << np.uint64(32)) | p["lo"].astype(np.uint64)
    assert (np.diff(key.astype(np.int64)) > 0).all()
    lo = g.debug("aabb_min", np.float32).reshape(-1, 4); hi = g.debug("aabb_max", np.float32).reshape(-1, 4)
    a, b = p["lo"].astype(np.int64), p["hi"].astype(np.int64)
    assert ((hi[a, :3] > lo[b, :3]) & (hi[b, :3] > lo[a, :3])).all()
    v = g.constraints_view()
    n = g.contacts.count
    srt = g.debug("sorted", np.uint32).astype(np.int64)
    tags, feats = g.contact_tags[:n][srt], g.contact_features[:n][srt]
    k1 = (tags >> np.uint64(32)).astype(np.int64); k2 = (tags & np.uint64(0xffffffff)).astype(np.int64)
    order_ok = (np.diff(k1) > 0) | ((np.diff(k1) == 0) & ((np.diff(k2) > 0) | ((np.diff(k2) == 0) & (np.diff(feats.astype(np.int64)) >= 0))))
    assert order_ok.all()
    batch = v["batch_of_contact"].astype(np.int64)
    bodies = g.contact_bodies[:n]
    for col in ("a", "b"):
        body = bodies[col].astype(np.int64)
        m = body != 0
        pairs = np.unique(np.stack([batch[m], body[m]], 1), axis=0)
        assert len(pairs) == m.sum() or col == "b"   # a body appears at most once per batch on each side
    allb = np.concatenate([np.stack([batch, bodies["a"].astype(np.int64)], 1), np.stack([batch, bodies["b"].astype(np.int64)], 1)])
    allb = allb[allb[:, 1] != 0]
    assert len(np.unique(allb, axis=0)) == len(allb), "a batch holds two contacts of one body"


def test_reference_own_test_program_on_the_gpu_dropin():
    """The reference's tests/main.cpp, compiled UNMODIFIED against nudge.h and linked against nudge_b200's namespace-nudge drop-in
    (oracle/_ref/ref_tests_on_gpu, built by oracle/Makefile), must print "All tests passed." — its six known-answer tests
    (20k collide() calls: contact counts 4 / 8 / 3 / 1 / 2, tag algebra, tests/main.cpp:130-1002) on the CUDA path."""
    import subprocess
    exe = os.path.join(os.path.dirname(G.HERE), "oracle", "_ref", "ref_tests_on_gpu")
    if not os.path.exists(exe):
        pytest.skip("oracle/_ref/ref_tests_on_gpu not built (needs /root/reference in the build container)")
    out = subprocess.run([exe], capture_output=True, text=True, timeout=900)
    assert out.returncode == 0 and "All tests passed." in out.stdout, out.stdout[-2000:] + out.stderr[-2000:]


def test_dropin_nudge_h_calls_equal_reference_on_a_trajectory():
    """Same Python harness, same nudge.h calls (uint16 layout, host pointers): reference CPU library vs the GPU drop-in, bit for bit."""
    from oracle import pyref
    if not os.path.exists(os.path.join(os.path.dirname(G.HERE), "oracle", "_ref", "libnudge_gpu_shim.so")):
        pytest.skip("oracle/_ref/libnudge_gpu_shim.so not built")
    s = scenes.demo_scene(200, 200, iterations=8, spread=3.0, height=30.0)
    r = pyref.RefSim(s); g = pyref.RefSim(s, gpu_dropin=True)
    for k in range(30):
        r.step_staged(); g.step_staged()
        assert r.contacts.count == g.contacts.count and r.cache.count == g.cache.count, "step %d" % k
        rv, gv = r.contacts_view(), g.contacts_view()
        for key in ("data", "bodies", "tags", "sleeping", "active"):
            assert np.array_equal(rv[key].view(np.uint8), gv[key].view(np.uint8)), "contacts.%s differs at step %d" % (key, k)
        assert np.array_equal(r.transforms.view(np.uint8), g.transforms.view(np.uint8)), "transforms differ at step %d" % k
        assert np.array_equal(r.momentum.view(np.uint8), g.momentum.view(np.uint8)), "momentum differs at step %d" % k
        assert np.array_equal(r.idle, g.idle)
        rc, gc = r.cache_view(), g.cache_view()
        assert np.array_equal(rc["tags"], gc["tags"]) and np.array_equal(rc["data"].view(np.uint8), gc["data"].view(np.uint8)), "cache differs at step %d" % k


def test_pack_unpack_momentum_kernels():
    import torch
    s = scenes.box_drop(2000, iterations=4)
    g = nudge_b200.Sim(s)
    rng = np.random.default_rng(3)
    g.momentum["velocity"][:] = rng.normal(size=(s.n_bodies, 3)); g.momentum["angular_velocity"][:] = rng.normal(size=(s.n_bodies, 3))
    g.upload_bodies()
    idx = torch.from_numpy(rng.permutation(s.n_bodies)[:500].astype(np.int32)).cuda()
    out = torch.zeros((500, 8), dtype=torch.float32, device="cuda")
    g.pack_momentum(idx.data_ptr(), 500, out.data_ptr())
    torch.cuda.synchronize()
    rows = g.momentum.view(np.float32).reshape(-1, 8)
    assert np.array_equal(out.cpu().numpy(), rows[idx.cpu().numpy()])
    # scatter rows src[i] of a buffer into bodies dst[i]
    dst = torch.from_numpy(np.arange(100, 600, dtype=np.int32)).cuda()
    src = torch.from_numpy(rng.integers(0, 500, 500).astype(np.int32)).cuda()
    g.unpack_momentum(dst.data_ptr(), src.data_ptr(), 500, out.data_ptr())
    g.download_bodies()
    want = rows.copy(); want[100:600] = out.cpu().numpy()[src.cpu().numpy()]
    assert np.array_equal(g.momentum.view(np.float32).reshape(-1, 8), want)


def test_sharded_scene_two_ranks_gpu_equals_oracle_ranks():
    """world_size 2 over gloo, both ranks on cuda:0: the sharded algorithm is a deterministic function of the partition, so the CUDA
    ranks must reproduce the oracle ranks bit for bit (ghost exchange after the warm start and after every sweep, two re-partitions)."""
    from tests import shard_util
    a = shard_util.run_ranks(2, "gpu", steps=12, reshard_every=5, n_boxes=600)
    b = shard_util.run_ranks(2, "oracle", steps=12, reshard_every=5, n_boxes=600)
    for r in range(2):
        assert np.array_equal(a[r]["transforms"].view(np.uint8), b[r]["transforms"].view(np.uint8))
        assert np.array_equal(a[r]["momentum"]["velocity"], b[r]["momentum"]["velocity"])
        assert np.array_equal(a[r]["counts"], b[r]["counts"])


def test_sharded_peer_memory_exchange_equals_host_exchange():
    """The C++ host's peer transport (nb_shard_step: k_shard_push / k_shard_pull over CUDA-IPC mapped inboxes, the arrival-flag protocol,
    the exchange plan) against the host-side exchange of the same partition: identical transforms and velocities on every rank.
    Two processes share cuda:0 here (they time-slice while waiting for each other); bench.py repeats the check on real multi-GPU boxes."""
    from tests import shard_util
    a = shard_util.run_ranks(2, "gpu_peer", steps=8, reshard_every=4, n_boxes=500)
    b = shard_util.run_ranks(2, "gpu", steps=8, reshard_every=4, n_boxes=500)
    for r in range(2):
        assert np.array_equal(a[r]["transforms"].view(np.uint8), b[r]["transforms"].view(np.uint8))
        assert np.array_equal(a[r]["momentum"]["velocity"], b[r]["momentum"]["velocity"])
        assert np.array_equal(a[r]["counts"], b[r]["counts"])


def test_body_connections_join_islands():
    """BodyConnections only feed the island passes (nudge.cpp:3511-3575, 3799-3863): a sleeping body connected to an awake one stays active."""
    s = scenes.demo_scene(60, 0, iterations=4, spread=40.0, height=2.0, seed=9)   # far apart: no contacts between boxes
    rng = np.random.default_rng(1)
    pairs = rng.integers(1, s.n_bodies, (25, 2))
    s.connections = np.zeros(len(pairs), scenes.PAIR32); s.connections["a"] = pairs[:, 0]; s.connections["b"] = pairs[:, 1]
    s.idle[:] = 0xff
    s.idle[pairs[:5, 0]] = 0     # a few awake bodies keep their connected partners active
    o, g = _pair(s)
    _steps(o, g, 3)
    assert 0 < g.active.count < s.n_bodies - 1


def test_sharded_step_graph_rerecords_when_the_connection_count_changes():
    """nb_shard_step's graph is keyed on the connection count like nb_step's: a world-1 shard and nb_step on the same scene stay equal
    byte for byte when nb_upload_connections changes the count between steps (connections decide which bodies stay awake here)."""
    import ctypes
    import torch
    s = scenes.demo_scene(60, 0, iterations=4, spread=40.0, height=2.0, seed=9)   # far apart: no contacts between boxes
    rng = np.random.default_rng(1)
    pairs = rng.integers(1, s.n_bodies, (25, 2))
    s.connections = np.zeros(len(pairs), scenes.PAIR32); s.connections["a"] = pairs[:, 0]; s.connections["b"] = pairs[:, 1]
    s.idle[:] = 0xff
    s.idle[pairs[:5, 0]] = 0     # the connections keep these bodies' partners awake
    sa, sb = torch.cuda.Stream(), torch.cuda.Stream()
    a = nudge_b200.Sim(s, stream=sa.cuda_stream)                  # nb_step
    b = nudge_b200.Sim(s, stream=sb.cuda_stream)                  # nb_shard_step, one rank, empty plan
    b.shard_create(0, 1, None, 1, 1)
    for n in (0, len(pairs)):
        for x in (a, b):
            x.conn.count = n
            x._ck(x.lib.nb_upload_connections(x.ctx, ctypes.byref(x.conn), x.stream), "nb_upload_connections")
        for _ in range(3):
            a.step(); b.shard_step("peer")
        a.download_bodies(); b.download_bodies()
        for name in ("transforms", "momentum", "idle"):
            assert getattr(a, name).tobytes() == getattr(b, name).tobytes(), "%s differs with %d connections" % (name, n)
    assert a.debug_scalar("graph_active") == 1 and b.shard_graph_active()
    assert a.counts().overflow == 0 and b.counts().overflow == 0


def test_config2_mixed_box_sphere_stack():
    """BASELINE configs[2] shape (50/50 box/sphere lattice stack, 16 iterations) at 20k bodies: settle on the GPU, then one step bit-exact vs the oracle."""
    s = scenes.mixed_stack(20000, iterations=16)
    o, g = _pair(s)
    for _ in range(150):
        g.step()
    assert g.counts().overflow == 0
    sync_oracle_from_gpu(o, g)
    _steps(o, g, 1)


def test_config4_brick_wall():
    """BASELINE configs[4] shape (running-bond wall of identical bricks: equal volumes, many 8-point manifolds, 20 iterations) at 20k bricks."""
    s = scenes.brick_wall(20000, iterations=20)
    o, g = _pair(s)
    for _ in range(60):
        g.step()
    assert g.counts().overflow == 0
    sync_oracle_from_gpu(o, g)
    _steps(o, g, 1)


def test_config3_one_million_boxes_runs_and_keeps_invariants():
    """BASELINE configs[3] size on ONE GPU: 1,048,576 boxes.  Too large for the CPU oracle in a test; checks capacity, that the pair list is
    sorted/unique, that every contact's bodies are a broadphase pair, and that nothing falls through the ground."""
    s = scenes.box_drop(1 << 20, iterations=8)
    g = nudge_b200.Sim(s, debug=True)
    for _ in range(40):
        g.step()
    c = g.counts()
    assert c.overflow == 0 and c.active == s.n_bodies - 1
    g.collide(); g.download_contacts()
    p = g.pairs_view()
    key = (p["hi"].astype(np.uint64) << np.uint64(32)) | p["lo"].astype(np.uint64)
    assert (np.diff(key.astype(np.int64)) > 0).all()
    n = g.contacts.count
    b = g.contact_bodies[:n]
    pk = np.minimum(b["a"], b["b"]).astype(np.uint64) << np.uint64(32) | np.maximum(b["a"], b["b"]).astype(np.uint64)
    allp = np.minimum(p["hi"], p["lo"]).astype(np.uint64) << np.uint64(32) | np.maximum(p["hi"], p["lo"]).astype(np.uint64)   # collider k sits on body k here
    assert np.isin(pk, allp).all()
    g.download_bodies()
    assert np.isfinite(g.transforms["position"]).all() and g.transforms["position"][1:, 1].min() > -1.0


def test_nb_step_graph_replay_equals_staged_calls_and_oracle():
    """nb_step on a capturable stream (CUDA graph replay, warm start fused into the first solver launch) against the seven stage
    calls on the default stream and against the oracle: same bits after 25 steps."""
    import torch
    from oracle import pyoracle
    scene = scenes.demo_scene(600, 600)
    side = torch.cuda.Stream()
    a = nudge_b200.Sim(scene)                                 # stage calls, default stream
    b = nudge_b200.Sim(scene, stream=side.cuda_stream)        # nb_step -> graph
    o = pyoracle.OracleSim(scene, contact_capacity=a.cap)
    for _ in range(25):
        a.step_staged(); b.step(); o.step()
    a.download_bodies(); b.download_bodies()
    launches_per_step = b.launch_count() / 25.0
    assert launches_per_step > 10
    for name in ("transforms", "momentum", "idle"):
        x, y, z = getattr(a, name), getattr(b, name), getattr(o, name)
        assert x.tobytes() == y.tobytes(), name
        assert x.tobytes() == z.tobytes(), name
    assert b.counts().overflow == 0 and a.counts().contacts == b.counts().contacts > 0


def test_hub_body_spills_the_scheduler_list_and_overflow_is_reported_not_hung():
    """ADVICE r1: one dynamic body with more contacts than the batch scheduler's on-chip slot list holds (16 buckets x 511 slots) used to
    leave a partial schedule behind and the dataflow solver waited forever.  Now (a) the list spills to global memory - the reference
    has no limit there - and the scene runs bit-identically to the oracle, and (b) when the constraint rows cannot hold the resulting
    batches the schedule is published EMPTY, the step finishes and the overflow is reported (nb_counts.overflow & 4)."""
    s = scenes.hub_platform(55, iterations=4)      # 3025 boxes x 4 contacts on the platform's body: 756 mutually conflicting contacts per bucket
    o, g = _pair(s)
    _steps(o, g, 3)
    assert g.counts().contacts > 8176 + 16 and g.counts().overflow == 0
    # the same scene with room for the contacts but not for one batch per platform contact
    small = nudge_b200.Sim(s, contact_capacity=16000)
    small.step_staged()
    c = small.counts()
    assert c.contacts > 8176 + 16 and (c.overflow & 4) and c.batches == 0
    with pytest.raises(nudge_b200.NudgeError):
        small.download_contacts()
    small.step_staged()                            # and the next step runs (no stale spill state, no hang)
    assert small.counts().overflow & 4
    o2, g2 = _pair(scenes.hub_platform(30, iterations=4))     # a hub inside the on-chip list
    _steps(o2, g2, 3)


def test_two_simulations_on_two_streams_replay_cooperative_step_graphs_concurrently():
    """ADVICE r1: grid-synchronising kernels inside the replayed graph keep the cooperative attribute, so two contexts stepping on two
    streams of one device cannot dead-lock each other; both must equal a lone simulation."""
    import torch
    scene = scenes.demo_scene(400, 400)
    sa, sb, sc = torch.cuda.Stream(), torch.cuda.Stream(), torch.cuda.Stream()
    a = nudge_b200.Sim(scene, stream=sa.cuda_stream); b = nudge_b200.Sim(scene, stream=sb.cuda_stream); c = nudge_b200.Sim(scene, stream=sc.cuda_stream)
    for _ in range(20):
        c.step()
    a.step(); a.download_bodies(); b.step(); b.download_bodies()      # one step each, alone: records the graphs
    assert a.debug_scalar("graph_active") == 1 and b.debug_scalar("graph_active") == 1
    for _ in range(19):
        a.step(); b.step()          # asynchronous: the two graphs are in flight together
    for x in (a, b, c):
        x.download_bodies()
    assert a.transforms.tobytes() == c.transforms.tobytes() and b.transforms.tobytes() == c.transforms.tobytes()


def test_headless_application_loop_on_the_dropin_equals_the_reference():
    """oracle/headless_example.cpp — an application loop over nudge.h in the shape of example/main.cpp:274-328, with the user's gravity
    loop on the host between the calls — linked with the reference's nudge.cpp (headless_ref) and with the GPU drop-in (headless_gpu):
    identical transform hashes after 120 steps, for one world and for two worlds stepped concurrently from two threads (one device
    context per world; the reference is re-entrant on disjoint data)."""
    import subprocess
    d = os.path.join(os.path.dirname(G.HERE), "oracle", "_ref")
    if not (os.path.exists(os.path.join(d, "headless_ref")) and os.path.exists(os.path.join(d, "headless_gpu"))):
        pytest.skip("oracle/_ref/headless_* not built (needs /root/reference in the build container)")
    for args in (["300", "300", "120", "8"], ["150", "150", "60", "8", "2"]):
        ref = subprocess.run([os.path.join(d, "headless_ref")] + args, capture_output=True, text=True, timeout=600)
        gpu = subprocess.run([os.path.join(d, "headless_gpu")] + args, capture_output=True, text=True, timeout=600)
        assert ref.returncode == 0 and gpu.returncode == 0, gpu.stdout + gpu.stderr
        worlds = lambda out: [l for l in out.splitlines() if l.startswith("world")]
        assert worlds(ref.stdout) == worlds(gpu.stdout) and len(worlds(ref.stdout)) == (2 if len(args) == 5 else 1), ref.stdout + gpu.stdout


@pytest.mark.parametrize("name", ["config2_mixed_256k", "config4_bricks_256k"])
def test_full_size_configs_2_and_4_one_step_parity(name):
    """BASELINE configs[2] (262,144 mixed boxes/spheres, 16 iterations) and configs[4] (262,144-brick wall, 20 iterations) at FULL size:
    settle on the GPU, then one complete step bit-exact against the widened CPU oracle from identical state (every stage compared:
    pair list, contacts, tag order, schedule, rows, momentum after all sweeps, cache, transforms)."""
    s = scenes.mixed_stack(262144, iterations=16) if name.startswith("config2") else scenes.brick_wall(262144, iterations=20)
    o, g = _pair(s)
    for _ in range(40):
        g.step()
    assert g.counts().overflow == 0
    sync_oracle_from_gpu(o, g)
    _steps(o, g, 1, individually=False)


def _pin_bodies(sim):
    import torch
    from nudge_b200 import abi
    keep = {}
    for name in ("transforms", "properties", "momentum", "idle"):
        a = getattr(sim, name)
        t = torch.empty(max(a.nbytes, 1), dtype=torch.uint8, pin_memory=True)
        v = t.numpy()[:a.nbytes].view(a.dtype)
        v[:] = a
        keep[name] = t; setattr(sim, name, v)
    sim.bodies = abi.BodyData(abi.ptr(sim.transforms), abi.ptr(sim.properties), abi.ptr(sim.momentum), abi.ptr(sim.idle), len(sim.transforms))
    return keep


def test_upload_step_download_with_the_side_copy_equals_single_stream_and_oracle(monkeypatch):
    """The end-to-end loop an application with host-side state runs (nb_upload_bodies + nb_step + nb_download_bodies every step, host
    edits in between): nb_upload_bodies sends momentum and properties on the library's copy stream so they travel under `collide`, and
    the captured step waits for them through an event-wait node.  Same bits as the same loop with NB_COPY_OVERLAP=0 (one stream), as
    the stage calls, and as the oracle fed the same edits."""
    import torch
    from oracle import pyoracle
    scene = scenes.demo_scene(500, 400, iterations=6, spread=4.0, height=30.0)
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    a = nudge_b200.Sim(scene, stream=s1.cuda_stream)               # side copy + graph replay
    monkeypatch.setenv("NB_COPY_OVERLAP", "0")
    b = nudge_b200.Sim(scene, stream=s2.cuda_stream)               # everything on the caller's stream
    monkeypatch.delenv("NB_COPY_OVERLAP")
    c = nudge_b200.Sim(scene, stream=s1.cuda_stream)               # side copy, stage calls (host-side join)
    o = pyoracle.OracleSim(scene, contact_capacity=a.cap)
    keep = [_pin_bodies(x) for x in (a, b, c)]
    rng = np.random.default_rng(3)
    for k in range(12):
        kick = rng.integers(1, scene.n_bodies, 40)
        dv = rng.normal(size=(40, 3)).astype(np.float32)
        for x in (a, b, c, o):
            x.momentum["velocity"][kick] += dv                     # the application's own code between two steps
            x.idle[kick] = 0
        for x in (a, b, c):
            x.upload_bodies()
        a.step(); b.step(); c.step_staged(); o.step()
        for x in (a, b, c):
            x.download_bodies()
        for name in ("transforms", "momentum", "idle"):
            assert getattr(a, name).tobytes() == getattr(o, name).tobytes(), "%s differs from the oracle at step %d" % (name, k)
            assert getattr(a, name).tobytes() == getattr(b, name).tobytes() == getattr(c, name).tobytes(), "%s differs between the upload paths at step %d" % (name, k)
    assert a.counts().overflow == 0 and a.counts().contacts > 0
    del keep
