"""Collider tags as applications assign them, on the GPU (tests/tag_cases.py builds the scenes):

  - monotone relabelling (no tag comparison changes) at every width of read_sort's key layouts: the run equals the dense-tag twin bit for
    bit at every stage, with every contact, cache and sleeping-pair tag mapped, through the stage calls and through nb_step's graph;
  - permuted and shared tags against the CPU oracle at every stage;
  - custom contacts uploaded with nb_upload_contacts whose tags no collider carries, through the C ABI against the oracle and through the
    nudge.h drop-in against the reference;
  - the sensor-overlap orientation of two colliders with equal tags, and a state file at 32 tag bits."""
import ctypes as C
import os
import subprocess
import tempfile
import numpy as np
import pytest
import nudge_b200
from nudge_b200 import scenes
from tests import tag_cases as T
from tests.gpu_util import side_stream, fnv1a
from tests.parity_util import Report, compare_oracle_gpu_step, sync_oracle_from_gpu

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HIGH32 = (0xffffffff, 0xfffffff0, 0x80000001, 0x12345678)   # custom-contact tags far beyond any collider's


def _sleepy_scene():
    return scenes.demo_scene(120, 120, iterations=4, spread=6.0, height=6.0, seed=11)


def _pile():
    return scenes.demo_scene(100, 100, iterations=4, spread=2.0, height=20.0)


def _force_sleep(sims, n_bodies):
    sleepy = np.random.default_rng(5).random(n_bodies) < 0.8
    for s in sims:
        s.download_bodies()
        s.idle[sleepy] = 0xff
        s.momentum["velocity"][sleepy] = 0; s.momentum["angular_velocity"][sleepy] = 0
        s.upload_bodies()


def _upload_contacts(g):
    g._ck(g.lib.nb_upload_contacts(g.ctx, C.byref(g.contacts), None, g.stream), "nb_upload_contacts")


def _premise(g, bits, internal=True):
    tb = g.debug_scalar("tagbits")
    assert tb == bits, "tagbits %d, the case was built for %d" % (tb, bits)
    lay = T.layout(tb, internal)
    print("tagbits %d: %s layout, contact sort over %s bits" % (tb, lay, T.key_bits(tb, internal)))
    return lay


def _twin_step(a, b, m, rep):
    """One step of the dense-tag sim `a` and its relabelled twin `b` (tags through TagMap m), every stage compared."""
    a.collide(); b.collide()
    a.download_contacts(); b.download_contacts()
    va, vb = a.contacts_view(), b.contacts_view()
    if not rep.check("contact count", va["count"] == vb["count"], "%d vs %d" % (va["count"], vb["count"])):
        return False
    for k in ("active", "data", "bodies", "features"):
        rep.eq(k, va[k], vb[k])
    rep.eq("tags (mapped)", m.pair(va["tags"]), vb["tags"]); rep.eq("sleeping (mapped)", m.pair(va["sleeping"]), vb["sleeping"])
    a.apply_gravity_damping(); b.apply_gravity_damping()
    a.read_cached_impulses(); b.read_cached_impulses()
    ia, ib = a.impulses_view(), b.impulses_view()
    rep.eq("sorted", ia["sorted"], ib["sorted"]); rep.eq("impulses", ia["data"], ib["data"])
    rep.eq("culled tags (mapped)", m.pair(ia["culled_tags"]), ib["culled_tags"]); rep.eq("culled data", ia["culled_data"], ib["culled_data"])
    a.setup_contact_constraints(); b.setup_contact_constraints()
    if va["count"]:
        ka, kb = a.constraints_view(), b.constraints_view()
        for k in ("contact", "rows", "states", "batch_of_contact", "slot_of_contact"):
            rep.eq(k, ka[k], kb[k])
    for it in range(int(a.scene.iterations)):
        a.apply_impulses(1); b.apply_impulses(1)
        a.download_bodies(); b.download_bodies()
        rep.eq("momentum sweep %d" % it, a.momentum, b.momentum)
    a.update_cached_impulses(); b.update_cached_impulses(); a.write_cached_impulses(); b.write_cached_impulses()
    a.download_cache(); b.download_cache()
    ca, cb = a.cache_view(), b.cache_view()
    rep.eq("cache tags (mapped)", m.pair(ca["tags"]), cb["tags"]); rep.eq("cache features", ca["features"], cb["features"]); rep.eq("cache data", ca["data"], cb["data"])
    a.advance(); b.advance()
    a.download_bodies(); b.download_bodies()
    for k in ("transforms", "momentum", "idle"):
        rep.eq(k, getattr(a, k), getattr(b, k))
    return rep.ok


def _read_launches(g):
    """Kernel launches of one nb_read_cached_impulses on the current contacts."""
    n0 = g.launch_count(); g.read_cached_impulses(); return g.launch_count() - n0


@pytest.mark.parametrize("bits", [3, 17, 22, 23, 24, 25, 31, 32])
def test_monotone_relabelling_is_bit_identical_at_every_layout(bits):
    """At 3 bits (8 colliders) the spread layout starts; 22 and 23 are its widest keys (61 and 63 bits); 24 fills a 64-bit key without the
    stretch, so the ground's contacts share one top-digit bucket; 25 and up take the two-pass sort, 32 with the largest tag 0xFFFFFFFF."""
    dense = scenes.demo_scene(4, 3, iterations=4, spread=0.8, height=4.0) if bits == 3 else _sleepy_scene()
    tagged, m = T.monotone(dense, bits, seed=bits)
    a, b = nudge_b200.Sim(dense, debug=True), nudge_b200.Sim(tagged, debug=True)
    lay = _premise(b, bits)
    a.collide(); b.collide()
    a.apply_gravity_damping(); b.apply_gravity_damping()
    extra = _read_launches(b) - _read_launches(a)
    assert T.layout(T.tagbits(dense)) == "spread"
    assert (extra > 0) == (lay == "two-pass"), "%s layout: %d more launches per read than the twin" % (lay, extra)
    a, b = nudge_b200.Sim(dense, debug=True), nudge_b200.Sim(tagged, debug=True)
    for i in range(40):
        rep = Report("%d bits step %d" % (bits, i))
        assert _twin_step(a, b, m, rep), str(rep)
    _force_sleep((a, b), dense.n_bodies)
    seen = 0
    for i in range(6):
        rep = Report("%d bits sleep %d" % (bits, i))
        assert _twin_step(a, b, m, rep), str(rep)
        seen = max(seen, b.contacts.sleeping_count)
    assert seen > 0 or bits == 3
    # nb_step's graph replay, from the same start
    ga, gb = nudge_b200.Sim(dense, stream=side_stream()), nudge_b200.Sim(tagged, stream=side_stream())
    for _ in range(30):
        ga.step(); gb.step()
    assert gb.debug_scalar("graph_active") == 1
    for x in (ga, gb):
        x.download_bodies(); x.download_cache()
    for k in ("transforms", "momentum", "idle"):
        assert getattr(ga, k).tobytes() == getattr(gb, k).tobytes(), k
    n = ga.cache.count
    assert n == gb.cache.count and np.array_equal(m.pair(ga.cache_tags[:n]), gb.cache_tags[:n])
    assert ga.cache_data[:n].tobytes() == gb.cache_data[:n].tobytes()


_SETTLED = {}


def _settled_pile():
    if "s" not in _SETTLED:
        s = scenes.box_drop(65536, iterations=8)
        g = nudge_b200.Sim(s, stream=side_stream())
        for _ in range(700):
            g.step()
        assert g.counts().overflow == 0
        g.download_bodies(); g.download_cache()
        n = g.cache.count
        _SETTLED["s"] = (g.export_state(), g.cache_tags[:n].copy(), g.cache_features[:n].copy(), g.cache_data[:n].copy())
    return _SETTLED["s"]


@pytest.mark.parametrize("bits", [23, 24, 25, 32])
def test_settled_65k_pile_relabelled_from_identical_state(bits):
    """The 65,536-box pile of BASELINE config 1, settled; then the dense twin and the relabelled one from the same state and cache."""
    state, ct, cf, cd = _settled_pile()
    tagged, m = T.monotone(state, bits, seed=100 + bits)
    a, b = nudge_b200.Sim(state), nudge_b200.Sim(tagged)
    _premise(b, bits)
    for x, tags in ((a, ct), (b, m.pair(ct))):
        n = len(tags)
        x.cache_tags[:n] = tags; x.cache_features[:n] = cf; x.cache_data[:n] = cd; x.cache.count = n
        x.upload_cache()
    for i in range(3):
        rep = Report("65k %d bits step %d" % (bits, i))
        assert _twin_step(a, b, m, rep), str(rep)
    assert b.counts().overflow == 0 and b.counts().contacts > 0


def _pair(scene):
    from oracle import pyoracle
    o = pyoracle.OracleSim(scene)
    g = nudge_b200.Sim(scene, contact_capacity=o.cap, debug=True)
    return o, g


@pytest.mark.parametrize("case", ["permuted", "permuted_sleeping", "shared_compound"])
def test_permuted_and_shared_tags_equal_the_oracle_at_every_stage(case):
    if case == "permuted":
        s = T.permuted(_pile(), seed=3)[0]
    elif case == "permuted_sleeping":
        s = T.permuted(_sleepy_scene(), seed=5, max_tag=0xffffffff)[0]
    else:
        s = T.shared(T.compound(_pile(), np.arange(1, 101, 3)))
    o, g = _pair(s)
    equal = 0
    for i in range(47 if case == "permuted_sleeping" else 20):
        if i == 40:
            _force_sleep((g,), s.n_bodies)
            g.download_bodies(); o.idle[:] = g.idle; o.momentum[:] = g.momentum
        rep = Report("%s step %d" % (case, i))
        assert compare_oracle_gpu_step(o, g, rep), str(rep)
        equal = max(equal, T.equal_tag_contacts(g.contact_tags[:g.contacts.count]))
    assert case != "shared_compound" or equal > 0


def test_permuted_tags_settled_65k_pile_one_step_against_the_oracle():
    state, ct, cf, cd = _settled_pile()
    tagged, m = T.permuted(state, seed=9, max_tag=0xffffffff)
    o, g = _pair(tagged)
    n = len(ct)
    tags = m.pair(ct)
    order = np.lexsort((cf, tags))   # the cache is ordered by (tag, feature); a permutation of the tags reorders it
    g.cache_tags[:n] = tags[order]; g.cache_features[:n] = cf[order]; g.cache_data[:n] = cd[order]; g.cache.count = n
    g.upload_cache()
    sync_oracle_from_gpu(o, g)
    _premise(g, 32)
    rep = Report("65k permuted")
    assert compare_oracle_gpu_step(o, g, rep, sweeps_individually=False), str(rep)


def test_custom_contacts_with_any_uint32_tags_equal_the_oracle():
    """nb_upload_contacts after nb_collide with contacts appended whose tags reach 0xFFFFFFFF and whose feature words are arbitrary,
    against body 0 and between awake bodies: every stage equals the oracle given the same rows, for several steps (the cache carries the
    custom entries from step to step)."""
    s = _pile()
    o, g = _pair(s)
    step = [0]

    def add(o, g):
        rows = T.custom_contacts(o, step[0], HIGH32, seed=1)
        assert len(rows)
        T.append_wide(o, rows); T.append_wide(g, rows)
        _upload_contacts(g)
    for i in range(12):
        step[0] = i
        rep = Report("custom contacts step %d" % i)
        assert compare_oracle_gpu_step(o, g, rep, after_collide=add), str(rep)
    g.download_cache()
    assert (g.cache_tags[:g.cache.count] >> np.uint64(32) >= np.uint64(0x12345676)).any()


def test_custom_contacts_through_the_dropin_equal_the_reference():
    """The reference's own hook (example/main.cpp:288) on the nudge.h drop-in: a 3,072-collider scene (12 tag bits) with custom contacts of
    tag 0xFFFF inserted between collide and read_cached_impulses, against the reference, byte for byte for 30 steps."""
    from oracle import pyref
    if not os.path.exists(os.path.join(ROOT, "oracle", "_ref", "libnudge_gpu_shim.so")):
        pytest.skip("oracle/_ref/libnudge_gpu_shim.so not built")
    s = scenes.demo_scene(1535, 1536, iterations=4, spread=20.0, height=60.0)
    assert s.n_colliders == 3072 and T.tagbits(s) == 12
    r, g = pyref.RefSim(s), pyref.RefSim(s, gpu_dropin=True)
    for k in range(30):
        for x in (r, g):
            x.collide()
        rows = T.custom_contacts(r, k, (0xffff, 0xfff0, 0xf00f), seed=2)
        for x in (r, g):
            T.append_ref(x, rows)
            x.apply_gravity_damping(); x.read_cached_impulses(); x.setup_contact_constraints()
            for _ in range(int(s.iterations)):
                x.apply_impulses()
            x.update_cached_impulses(); x.write_cached_impulses(); x.advance()
        assert r.contacts.count == g.contacts.count and r.cache.count == g.cache.count, "step %d" % k
        rv, gv = r.contacts_view(), g.contacts_view()
        for key in ("data", "bodies", "tags", "sleeping", "active"):
            assert rv[key].tobytes() == gv[key].tobytes(), "contacts.%s differs at step %d" % (key, k)
        rc, gc = r.cache_view(), g.cache_view()
        assert rc["tags"].tobytes() == gc["tags"].tobytes() and rc["data"].tobytes() == gc["data"].tobytes(), "cache differs at step %d" % k
        assert r.momentum.tobytes() == g.momentum.tobytes(), "momentum differs at step %d" % k
        assert r.transforms.tobytes() == g.transforms.tobytes(), "transforms differ at step %d" % k


def test_sensor_overlap_of_equal_tags_puts_the_lower_body_first():
    """A sensor collider given the tag of a collider it overlaps: sensors never reach the contacts, so the physics is the twin's; the overlap
    list is the twin's with that tag mapped, and for the equal-tag entry body_a is the lower body."""
    from tests.sensor_ref import add_sensors
    s = scenes.demo_scene(100, 100, iterations=4, spread=3.0, height=10.0, seed=21)
    s.transforms["position"][1:, 1] -= 6.0
    dense = add_sensors(s, zones=[((0.0, -8.5, 0.0), (2.0, 1.5, 2.0))], proximity=(4, 50), falling=(7, 77))
    a = nudge_b200.Sim(dense)
    hit = None
    for i in range(40):
        a.step_staged()
        ov = a.sensor_overlaps()
        if len(ov):
            hit = (i, ov[0]); break
    assert hit is not None
    lo, hi = int(hit[1]["tags"] & 0xffffffff), int(hit[1]["tags"] >> 32)   # dense tags are collider indices here
    sens, other = (lo, hi) if dense.sensors[lo] else (hi, lo)
    f = np.arange(dense.n_colliders, dtype=np.uint64); f[sens] = other
    m = T.TagMap(f)
    tagged = m.apply(dense)
    a, b = nudge_b200.Sim(dense), nudge_b200.Sim(tagged)
    body = np.concatenate([dense.box_transforms["body"], dense.sphere_transforms["body"]]).astype(np.uint32)
    equal = False
    for i in range(hit[0] + 3):
        a.step_staged(); b.step_staged()
        want = a.sensor_overlaps()
        t = want["tags"]
        ta, tb = t & T.MASK32, t >> T.S32
        fa, fb = m.tag(ta), m.tag(tb)
        exp = np.zeros(len(want), scenes.SENSOR_OVERLAP)
        exp["tags"] = np.minimum(fa, fb) | (np.maximum(fa, fb) << T.S32)
        ba, bb = body[ta.astype(np.int64)], body[tb.astype(np.int64)]
        first = np.where(fa != fb, fa < fb, ba < bb)
        exp["body_a"] = np.where(first, ba, bb); exp["body_b"] = np.where(first, bb, ba)
        exp = exp[np.argsort(exp["tags"], kind="stable")]
        got = b.sensor_overlaps()
        assert got.tobytes() == exp.tobytes(), "step %d" % i
        equal |= bool(((got["tags"] & T.MASK32) == (got["tags"] >> T.S32)).any())
    assert equal
    a.download_bodies(); b.download_bodies()
    assert a.transforms.tobytes() == b.transforms.tobytes()


def test_state_file_at_32_tag_bits_continues_and_replays():
    tagged, m = T.monotone(_sleepy_scene(), 32, seed=32)
    st = side_stream()
    g = nudge_b200.Sim(tagged, stream=st)
    for _ in range(30):
        g.step()
    d = tempfile.mkdtemp(prefix="nb_tags_")
    p = os.path.join(d, "s.bin")
    g.save_state(p)
    h = nudge_b200.Sim(_sleepy_scene(), stream=st)
    h.load_state(p)
    assert h.debug_scalar("tagbits") == 32
    for _ in range(10):
        g.step(); h.step()
    for x in (g, h):
        x.download_bodies(); x.download_cache()
    for k in ("transforms", "momentum", "idle"):
        assert getattr(g, k).tobytes() == getattr(h, k).tobytes(), k
    n = g.cache.count
    assert n == h.cache.count and g.cache_tags[:n].tobytes() == h.cache_tags[:n].tobytes() and (g.cache_tags[:n] >> T.S32 > 0xffffff).any()
    exe = os.path.join(ROOT, "tools", "bin", "nb_replay")
    out = subprocess.run([exe, p, "--steps", "10", "--iterations", str(tagged.iterations)], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stdout + out.stderr
    last = out.stdout.strip().splitlines()[-1].split()
    assert int(last[last.index("xf") + 1], 16) == fnv1a(g.transforms.tobytes())
