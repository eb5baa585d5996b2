"""Collision filters on the device (nb_upload_collision_filters, DESIGN.md section 8.6) against the filtered restatement of the CPU oracle
(tests/filter_ref.py), bit for bit: every stage of a mixed scene with three categories and a ground some spheres ignore, an all-pass or removed table against a plain context,
the connected opt-out on a chain of overlapping jointed links, graph replay while the table changes, END events of a pair that becomes
rejected, throughput mode, state files of version 1 and 2 with the replay tool, and the argument errors."""
import ctypes, os, struct, subprocess, tempfile
import numpy as np
import pytest
import nudge_b200
from nudge_b200 import scenes
from tests.parity_util import Report, compare_oracle_gpu_step, sync_oracle_from_gpu
from tests.test_gpu_rows import ball_joint_rows, _quat_rotate
from tests.gpu_util import fnv1a, side_stream, state_size

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NB_ERR_ARGUMENT = -3


def _oracle(scene):
    from tests.filter_ref import FilteredOracleSim
    return FilteredOracleSim(scene)


def _filters(n, nboxes, seed=4):
    """Categories 1, 2, 4 at random; 2 and 4 ignore each other; the ground (collider 0) is category 1 and a fifth of the spheres do
    not collide with it (they fall through: the ground is a large collider, so this goes through k_large_pairs)."""
    rng = np.random.default_rng(seed)
    cat = (1 << rng.integers(0, 3, n)).astype(np.uint16)
    mask = np.full(n, 7, np.uint16)
    mask[cat == 2] = 3; mask[cat == 4] = 5
    cat[0] = 1; mask[0] = 7
    sph = np.arange(nboxes, n)
    mask[sph[rng.random(len(sph)) < 0.2]] &= 6
    f = np.zeros(n, scenes.FILTER); f["category"] = cat; f["mask"] = mask
    return f


def _mixed(seed=11):
    s = scenes.demo_scene(120, 120, iterations=4, spread=3.0, height=12.0, seed=seed)
    s.collision_filters = _filters(s.n_colliders, s.n_boxes)
    return s


def _passes(f, a, b):
    return bool(f["category"][a] & f["mask"][b]) and bool(f["category"][b] & f["mask"][a])


def _collider_of_tag(s):
    return {int(t): i for i, t in enumerate(np.concatenate([s.box_tags, s.sphere_tags]))}


def _contact_colliders(g, s):
    g.download_contacts()
    m = _collider_of_tag(s)
    tags = np.unique(g.contact_tags[:g.contacts.count])
    return [(m[int(t) & 0xffffffff], m[int(t) >> 32]) for t in tags]


def _same_state(a, b, what):
    a.download_bodies(); b.download_bodies(); a.download_cache(); b.download_cache()
    for name in ("transforms", "momentum", "idle"):
        assert getattr(a, name).tobytes() == getattr(b, name).tobytes(), "%s: %s" % (what, name)
    n = a.cache.count
    assert n == b.cache.count and a.cache_tags[:n].tobytes() == b.cache_tags[:n].tobytes() and a.cache_data[:n].tobytes() == b.cache_data[:n].tobytes(), what


def test_bit_parity_with_the_filtered_oracle_stage_by_stage():
    s = _mixed()
    o = _oracle(s)
    g = nudge_b200.Sim(s, contact_capacity=o.cap, debug=True)
    assert g.lut_model_exact()
    from oracle import pyoracle
    plain = pyoracle.OracleSim(scenes.demo_scene(120, 120, iterations=4, spread=3.0, height=12.0, seed=11))
    for i in range(30):
        if i % 10 == 0:   # the unfiltered pair count of the same state
            sync_oracle_from_gpu(plain, g); plain.collide()
            unfiltered = int(plain.lib.nbo_last_pair_count())
        rep = Report("filtered step %d" % i)
        assert compare_oracle_gpu_step(o, g, rep), str(rep)
        if i % 10 == 0:
            assert unfiltered > g.counts().pairs > 0, (unfiltered, g.counts().pairs)
    f = s.collision_filters
    assert all(_passes(f, a, b) for a, b in _contact_colliders(g, s))
    sleepy = np.ones(s.n_bodies, bool)   # the pile is one island: put it to sleep, then wake it with one body
    for x in (o, g):
        x.idle[sleepy] = 0xff
        x.momentum["velocity"][sleepy] = 0; x.momentum["angular_velocity"][sleepy] = 0
    g.upload_bodies()
    seen = 0
    for i in range(6):
        if i == 3:
            for x in (o, g):
                x.idle[3] = 0
            g.upload_bodies()
        rep = Report("filtered sleep %d" % i)
        assert compare_oracle_gpu_step(o, g, rep), str(rep)
        seen = max(seen, g.contacts.sleeping_count)
    assert seen > 0


def test_all_pass_and_removed_tables_equal_a_plain_context():
    s = scenes.demo_scene(150, 150, iterations=4, spread=3.0, height=15.0, seed=3)
    plain, passing, removed = (nudge_b200.Sim(s, stream=side_stream()) for _ in range(3))
    allpass = np.zeros(s.n_colliders, scenes.FILTER); allpass["category"] = 0xffff; allpass["mask"] = 0xffff
    passing.upload_collision_filters(allpass)
    removed.upload_collision_filters(_filters(s.n_colliders, s.n_boxes)); removed.upload_collision_filters(None)
    for i in range(40):
        used = []
        for x in (plain, passing, removed):
            before = x.launch_count()
            x.step_staged() if i < 10 else x.step()
            used.append(x.launch_count() - before)
        assert used[0] == used[1] == used[2], (i, used)
    for x in (passing, removed):
        _same_state(plain, x, "after 40 steps")
        assert x.counts().pairs == plain.counts().pairs > 0
    assert plain.debug_scalar("graph_active") == 1 and passing.debug_scalar("graph_active") == 1


def _chain(links, half_length):
    """The hanging chain of test_gpu_rows, links of half length `half_length` jointed 0.5 from their centres: > 0.5 overlaps at the joints."""
    s = scenes.demo_scene(links + 60, 0, iterations=12, spread=3.0, height=6.0, seed=5)
    s.box_data["size"][1:links + 1] = (0.2, half_length, 0.2)
    s.properties[1:links + 1] = scenes._box_props(s.box_data["size"][1:links + 1])
    top = np.array([6.0, 8.0, 0.0])
    for k in range(links):
        s.transforms["position"][1 + k] = top + np.array([0.5 + 1.0 * k, 0.0, 0.0])
        s.transforms["rotation"][1 + k] = (0.0, 0.0, np.sin(np.pi / 4), np.cos(np.pi / 4))
    s.connections = np.zeros(links - 1, scenes.PAIR32); s.connections["a"] = 1 + np.arange(links - 1); s.connections["b"] = 2 + np.arange(links - 1)
    return s, top


def _chain_rows(g, links, top, dt):
    g.download_bodies()
    rows = [ball_joint_rows(g.transforms, 1, 0, (0.0, 0.5, 0.0), top, dt)]
    for k in range(1, links):
        rows.append(ball_joint_rows(g.transforms, 1 + k, k, (0.0, 0.5, 0.0), (0.0, -0.5, 0.0), dt))
    return np.concatenate(rows)


def _joint_error(g, links):
    g.download_bodies()
    worst = 0.0
    for k in range(1, links):
        wa = g.transforms["position"][1 + k] + _quat_rotate(g.transforms["rotation"][1 + k].astype(np.float64), np.array([0.0, 0.5, 0.0]))
        wb = g.transforms["position"][k] + _quat_rotate(g.transforms["rotation"][k].astype(np.float64), np.array([0.0, -0.5, 0.0]))
        worst = max(worst, float(np.linalg.norm(wa - wb)))
    return worst


def _connected_contacts(g, links):
    g.download_contacts()
    b = g.contact_bodies[:g.contacts.count]
    lo, hi = np.minimum(b["a"], b["b"]), np.maximum(b["a"], b["b"])
    return int(((lo >= 1) & (hi == lo + 1) & (hi <= links)).sum())


def test_connected_opt_out_lets_overlapping_jointed_links_hang_together():
    links = 10
    s, top = _chain(links, 0.6)
    o = _oracle(s); o.upload_collision_filters(None, scenes.FILTER_SKIP_CONNECTED)
    g = nudge_b200.Sim(s, contact_capacity=o.cap, debug=True)
    g.upload_collision_filters(None, scenes.FILTER_SKIP_CONNECTED)
    dt = float(s.time_step)
    worst, contacts = 0.0, 0
    for step in range(240):
        g.upload_constraint_rows(_chain_rows(g, links, top, dt))
        if step in (0, 120, 239):   # the collide stage from the same state equals the filtered oracle's
            sync_oracle_from_gpu(o, g)
            o.collide(); g.collide()
            g.download_contacts()
            oc, gc = o.contacts_view(), g.contacts_view()
            op, gp = o.pairs_view(), g.pairs_view()
            rep = Report("chain collide %d" % step)
            rep.eq("pairs.lo", op["lo"], gp["lo"]); rep.eq("pairs.hi", op["hi"], gp["hi"])
            for k in ("data", "bodies", "tags", "features", "sleeping", "active"):
                rep.eq(k, oc[k], gc[k])
            assert rep.ok, str(rep)
            g.apply_gravity_damping(); g.read_cached_impulses(); g.setup_contact_constraints(); g.apply_impulses(int(s.iterations))
            g.update_cached_impulses(); g.write_cached_impulses(); g.advance()
        else:
            g.step_staged()
        contacts += _connected_contacts(g, links)
        if step > 20:
            worst = max(worst, _joint_error(g, links))
    print("overlapping chain with NB_FILTER_SKIP_CONNECTED: worst joint error %.4f" % worst)
    assert contacts == 0
    assert worst < 0.04, worst
    assert np.isfinite(g.transforms["position"]).all() and g.counts().overflow == 0
    assert g.transforms["position"][links][1] < top[1] - 0.5 * links
    # without the flag the same links collide where they overlap
    h = nudge_b200.Sim(s)
    for step in range(5):
        h.upload_constraint_rows(_chain_rows(h, links, top, dt))
        h.step_staged()
        contacts += _connected_contacts(h, links)
    assert contacts > 0


def test_graph_replay_equals_staged_calls_while_the_table_changes():
    s = _mixed(seed=12)
    table = s.collision_filters
    s.collision_filters = None
    a = nudge_b200.Sim(s, stream=side_stream()); b = nudge_b200.Sim(s, stream=side_stream())
    other = _filters(s.n_colliders, s.n_boxes, seed=8)
    for i in range(40):
        if i in (10, 20, 30):
            f = {10: table, 20: other, 30: None}[i]
            a.upload_collision_filters(f); b.upload_collision_filters(f)
        a.step(); b.step_staged()
        if i % 5 == 4 or i in (10, 20, 30):
            _same_state(a, b, "step %d" % i)
        if 10 <= i < 30:
            f = table if i < 20 else other
            assert all(_passes(f, x, y) for x, y in _contact_colliders(a, s)), i
    assert a.debug_scalar("graph_active") == 1


def test_a_touching_pair_that_becomes_rejected_ends_once():
    from oracle import events_ref
    s = scenes.demo_scene(150, 150, iterations=4, spread=5.0, height=12.0, seed=4)
    o = _oracle(s); rec = events_ref.OracleEvents(o)
    g = nudge_b200.Sim(s, contact_capacity=o.cap, stream=side_stream())
    g.enable_contact_events(1 << 16)

    def same(what):
        want = rec.step(); g.step()
        got, dropped = g.contact_events()
        assert dropped == 0 and len(got) == len(want) and got.tobytes() == want.tobytes(), what
        return got
    for i in range(40):
        same("step %d" % i)
    g.download_cache()
    key = int(g.cache_tags[0])
    m = _collider_of_tag(s)
    a, b = m[key & 0xffffffff], m[key >> 32]
    f = np.zeros(s.n_colliders, scenes.FILTER); f["category"] = 0xffff; f["mask"] = 0xffff
    f[a] = (1, 0xfffd); f[b] = (2, 0xffff)                # only the pair (a, b) fails the rule
    g.upload_collision_filters(f); o.upload_collision_filters(f)
    got = same("the step after the upload")
    ends = got[(got["kind"] == scenes.CONTACT_END) & (got["tags"] == key)]
    assert len(ends) == 1
    g.download_cache()
    assert key not in set(int(t) for t in g.cache_tags[:g.cache.count])
    for i in range(5):
        got = same("later step %d" % i)
        assert key not in set(int(t) for t in got["tags"])


def test_throughput_mode_collides_like_parity_mode_and_never_joins_rejected_colliders():
    s = _mixed(seed=13)
    p = nudge_b200.Sim(s, debug=True); t = nudge_b200.Sim(s, debug=True)
    t.set_solver_mode("throughput")
    for _ in range(5):
        p.step_staged()
    p.download_bodies()
    t.transforms[:] = p.transforms; t.momentum[:] = p.momentum; t.idle[:] = p.idle
    t.upload_bodies()
    p.collide(); t.collide()
    for k, v in p.pairs_view().items():
        assert np.array_equal(v, t.pairs_view()[k]), k
    p.download_contacts(); t.download_contacts()
    pc, tc = p.contacts_view(), t.contacts_view()
    for k in ("data", "bodies", "tags", "features", "sleeping", "active"):
        assert pc[k].tobytes() == tc[k].tobytes(), k
    t.apply_gravity_damping(); t.read_cached_impulses(); t.setup_contact_constraints(); t.apply_impulses(int(s.iterations))
    t.update_cached_impulses(); t.write_cached_impulses(); t.advance()
    for _ in range(20):
        t.step_staged()
        assert all(_passes(s.collision_filters, a, b) for a, b in _contact_colliders(t, s))
    assert t.counts().contacts > 0


def test_filtered_state_saves_as_version_2_loads_and_replays():
    side = side_stream()
    s = _mixed(seed=14)
    s.connections = np.zeros(3, scenes.PAIR32); s.connections["a"] = (1, 5, 9); s.connections["b"] = (2, 6, 10)
    s.filter_flags = scenes.FILTER_SKIP_CONNECTED
    g = nudge_b200.Sim(s, stream=side)
    for _ in range(30):
        g.step()
    d = tempfile.mkdtemp(prefix="nb_filter_state_")
    p1, p2, p3 = (os.path.join(d, x) for x in ("a.bin", "b.bin", "plain.bin"))
    g.save_state(p1)
    raw = open(p1, "rb").read()
    version, = struct.unpack_from("<I", raw, 8); reserved = struct.unpack_from("<8I", raw, 36)
    assert version == 2 and reserved[0] == scenes.FILTER_SKIP_CONNECTED and reserved[1] == 1
    cache = struct.unpack_from("<I", raw, 28)[0]
    assert len(raw) == state_size(s.n_bodies, s.n_boxes, s.n_spheres, 3, cache, True)
    tail = raw[len(raw) - (4 * s.n_colliders + 15) // 16 * 16:][:4 * s.n_colliders]
    assert tail == s.collision_filters.tobytes()
    other = scenes.demo_scene(120, 120, iterations=4, seed=99); other.connections = np.zeros(3, scenes.PAIR32)
    h = nudge_b200.Sim(other, stream=side)
    h.load_state(p1)
    for _ in range(10):
        g.step(); h.step()
    _same_state(g, h, "loaded filtered state")
    exe = os.path.join(ROOT, "tools", "bin", "nb_replay")
    out = subprocess.run([exe, p1, "--steps", "10", "--iterations", str(int(s.iterations)), "--dump", p2], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stdout + out.stderr
    last = out.stdout.strip().splitlines()[-1].split()
    assert int(last[last.index("xf") + 1], 16) == fnv1a(g.transforms.tobytes())
    assert open(p2, "rb").read()[8:12] == struct.pack("<I", 2)
    # a version-1 load removes the table and the flags: the context steps like a plain one
    plain_scene = scenes.demo_scene(120, 120, iterations=4, spread=3.0, height=12.0, seed=14)
    plain = nudge_b200.Sim(plain_scene, stream=side)
    plain.save_state(p3)
    raw = open(p3, "rb").read()
    assert struct.unpack_from("<I", raw, 8)[0] == 1 and len(raw) == state_size(plain_scene.n_bodies, plain_scene.n_boxes, plain_scene.n_spheres, 0, 0, False)
    h.load_state(p3)
    for _ in range(5):
        h.step(); plain.step()
    _same_state(plain, h, "version-1 load after a filtered context")


def test_wrong_count_is_refused_and_the_table_follows_the_collider_count():
    s = scenes.demo_scene(40, 40, iterations=4, spread=2.0, height=6.0, seed=6)
    g = nudge_b200.Sim(s)
    n = s.n_colliders
    f = np.zeros(n, scenes.FILTER); f["category"] = 1; f["mask"] = 0   # nothing collides
    for bad in (n - 1, n + 1):
        r = g.lib.nb_upload_collision_filters(g.ctx, f.ctypes.data_as(ctypes.c_void_p), bad, 0, g.stream)
        assert r == NB_ERR_ARGUMENT
    g.collide(); assert g.counts().pairs > 0
    g.upload_collision_filters(f)
    g.collide(); assert g.counts().pairs == 0
    g._ck(g.lib.nb_upload_colliders(g.ctx, ctypes.byref(g.colliders), g.stream), "nb_upload_colliders")   # same count: kept
    g.collide(); assert g.counts().pairs == 0
    fewer = scenes.demo_scene(40, 39, iterations=4, spread=2.0, height=6.0, seed=6)
    g.reload(fewer)                                                     # another count: removed
    g.collide(); assert g.counts().pairs > 0
    r = g.lib.nb_upload_collision_filters(g.ctx, f.ctypes.data_as(ctypes.c_void_p), n, 0, g.stream)
    assert r == NB_ERR_ARGUMENT                                         # the old count no longer fits
