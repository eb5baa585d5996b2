"""Contact begin / end events (nb_enable_contact_events, nb_download_contact_events) against the restatement oracle/events_ref.py on the
CPU oracle, byte for byte, through nb_step's graph replay, the stage calls, throughput mode, small buffers, uploaded caches, a scene with
more than 50k contacts, and the sharded step's refusal."""
import ctypes
import numpy as np
import pytest
import nudge_b200
from nudge_b200 import scenes
from tests.parity_util import sync_oracle_from_gpu

pytestmark = pytest.mark.gpu
NB_ERR_CAPACITY, NB_ERR_ARGUMENT, NB_ERR_OVERFLOW = -2, -3, -4


def _oracle(scene):
    from oracle import pyoracle
    return pyoracle.OracleSim(scene)


def _recorder(o):
    from oracle import events_ref
    return events_ref.OracleEvents(o)


def _stream():
    import torch
    return torch.cuda.Stream().cuda_stream


def _sim(scene, o, stream=0, capacity=1 << 16):
    g = nudge_b200.Sim(scene, contact_capacity=o.cap, stream=stream)
    assert g.lut_model_exact(), "host CPU's rcpps/rsqrtps do not follow the LUT model: bit parity is not expected on this box"
    g.enable_contact_events(capacity)
    return g


def _same(got, want, what):
    assert len(got) == len(want), "%s: %d events, expected %d" % (what, len(got), len(want))
    bad = np.nonzero(got.view(np.uint8).reshape(-1, 80) != want.view(np.uint8).reshape(-1, 80))[0]
    assert len(bad) == 0, "%s: event %d differs: %r != %r" % (what, bad[0], got[bad[0]], want[bad[0]])


def _drain(g, capacity):
    """The raw call: (status, events, count, dropped)."""
    out = np.zeros(max(capacity, 1), scenes.CONTACT_EVENT)
    n = ctypes.c_uint32(0); d = ctypes.c_uint32(0)
    r = g.lib.nb_download_contact_events(g.ctx, out.ctypes.data_as(ctypes.c_void_p), capacity, ctypes.byref(n), ctypes.byref(d), g.stream)
    return r, out[:n.value].copy(), int(n.value), int(d.value)


def _falling():
    return scenes.demo_scene(150, 150, iterations=4, spread=5.0, height=12.0, seed=4)


def test_graph_replay_equals_restatement_and_late_drains_get_the_concatenation():
    s = _falling()
    o = _oracle(s); rec = _recorder(o)
    g = _sim(s, o, _stream()); late = _sim(s, o, _stream())
    kinds, want_late = set(), []
    for i in range(40):
        want = rec.step()
        g.step(); late.step()
        got, dropped = g.contact_events()
        _same(got, want, "step %d" % i)
        assert dropped == 0
        kinds |= set(int(k) for k in want["kind"])
        want_late.append(want)
        if i % 5 == 4:
            got, dropped = late.contact_events()
            _same(got, np.concatenate(want_late), "drain after step %d" % i)
            want_late = []
    assert kinds == {scenes.CONTACT_BEGIN, scenes.CONTACT_END}
    assert g.debug_scalar("graph_active") == 1 and g.counts().overflow == 0


def test_sleeping_pairs_do_not_end_and_a_kicked_subset_does():
    s = scenes.demo_scene(120, 120, iterations=4, spread=6.0, height=6.0, seed=11)
    o = _oracle(s); rec = _recorder(o)
    g = _sim(s, o)
    for i in range(40):
        want = rec.step(); g.step_staged()
        _same(g.contact_events()[0], want, "step %d" % i)
    g.download_bodies()
    sleepy = np.random.default_rng(5).random(s.n_bodies) < 0.8
    for x in (o, g):
        x.idle[sleepy] = 0xff
        x.momentum["velocity"][sleepy] = 0; x.momentum["angular_velocity"][sleepy] = 0
    g.upload_bodies()
    asleep = set()
    for i in range(6):
        want = rec.step(); g.step_staged()
        _same(g.contact_events()[0], want, "asleep step %d" % i)
        g.download_contacts()
        asleep |= set(int(t) for t in g.debug("culled_tags", np.uint64))
        ended = set(int(t) for t in want["tags"][want["kind"] == scenes.CONTACT_END])
        assert not (ended & asleep), "a sleeping pair ended"
    assert asleep, "no pair went to sleep"
    g.download_bodies()
    kick = np.nonzero(sleepy)[0][::4]
    for x in (o, g):
        x.idle[kick] = 0
        x.momentum["velocity"][kick, 1] = 6.0
    g.upload_bodies()
    ends = 0
    for i in range(6):
        want = rec.step(); g.step_staged()
        _same(g.contact_events()[0], want, "after the kick, step %d" % i)
        ends += int((want["kind"] == scenes.CONTACT_END).sum())
    assert ends > 0


def test_stage_calls_equal_graph_replay_and_throughput_mode_follows_the_contract():
    from oracle import events_ref
    s = _falling()
    o = _oracle(s)
    a = _sim(s, o, _stream()); b = _sim(s, o)
    for i in range(25):
        a.step(); b.step_staged()
        _same(a.contact_events()[0], b.contact_events()[0], "step %d" % i)
    t = _sim(s, o, _stream())
    t.set_solver_mode("throughput")
    t.enable_contact_events(1 << 16)
    fields = [f for f in scenes.CONTACT_EVENT.names if f != "impulse"]
    n_events = 0
    for i in range(25):
        t.download_cache(); old = t.cache_view()
        t.step()
        got, dropped = t.contact_events()
        t.download_contacts()
        cur = t.contacts_view()
        imp = t.debug("impulses", scenes.IMPULSE)["impulse"]
        want = events_ref.events(old["tags"], cur, imp, t.debug("culled_tags", np.uint64), i)
        assert len(got) == len(want) and dropped == 0
        for f in fields:
            assert got[f].tobytes() == want[f].tobytes(), "throughput step %d: %s differs" % (i, f)
        n_events += len(got)
    assert n_events > 0


def test_a_small_buffer_keeps_the_first_events_and_counts_the_rest():
    s = _falling()
    o = _oracle(s)
    big = _sim(s, o)
    small = _sim(s, o, capacity=7)
    full = []
    for _ in range(12):
        big.step_staged(); small.step_staged()
        full.append(big.contact_events()[0])
    full = np.concatenate(full)
    assert len(full) > 7
    r, _, n, d = _drain(small, 3)                 # host buffer smaller than what is stored: nothing is drained
    assert (r, n, d) == (NB_ERR_CAPACITY, 7, len(full) - 7)
    r, got, n, d = _drain(small, 7)
    assert r == NB_ERR_OVERFLOW and "dropped" in small.lib.nb_last_error(small.ctx).decode()
    _same(got, full[:7], "prefix")
    assert d == len(full) - 7
    r, got, n, d = _drain(small, 7)
    assert (r, n, d) == (0, 0, 0)
    big.step_staged(); small.step_staged()
    want = big.contact_events()[0]
    got, dropped = small.contact_events()
    _same(got, want[:7], "next step")
    assert dropped == max(0, len(want) - 7)
    r, _, _, _ = _drain(nudge_b200.Sim(s), 4)
    assert r == NB_ERR_ARGUMENT                   # never enabled


def test_launches_per_step_and_graph_rerecording():
    s = _falling()
    g = nudge_b200.Sim(s, stream=_stream())

    def per_step():
        g.step(); g.download_bodies()
        n0 = g.launch_count()
        g.step(); g.download_bodies()
        return g.launch_count() - n0

    base = per_step()
    g.enable_contact_events(0)
    assert per_step() == base and g.debug_scalar("graph_active") == 1
    g.enable_contact_events(1000)
    assert per_step() == base + 3 and g.debug_scalar("graph_active") == 1
    assert len(g.contact_events()[0]) > 0         # the re-recorded graph produces events
    g.enable_contact_events(10)                   # smaller: the buffer is reused, the graph still re-records (capacity is a launch argument)
    per_step()
    assert len(g.contact_events()[0]) <= 10
    g.enable_contact_events(0)
    assert per_step() == base and g.debug_scalar("graph_active") == 1
    n0 = g.launch_count(); g.step_staged(); staged = g.launch_count() - n0
    g.enable_contact_events(1000)
    n0 = g.launch_count(); g.step_staged()
    assert g.launch_count() - n0 == staged + 3


def test_an_uploaded_cache_counts_as_touching():
    s = _falling()
    o = _oracle(s)
    warm = nudge_b200.Sim(s, contact_capacity=o.cap)
    for _ in range(30):
        warm.step_staged()
    sync_oracle_from_gpu(o, warm)
    n = o.cache.count
    keys = np.unique(o.cache_tags[:n])
    assert len(keys) > 10
    keep = ~np.isin(o.cache_tags[:n], keys[::3])             # every third pair is forgotten: it begins again
    k = s.n_colliders
    fake = np.uint64(k + 1) | (np.uint64(k) << np.uint64(32))   # a pair of tags no collider has: it ends
    tags = np.concatenate([o.cache_tags[:n][keep], [fake]]); feats = np.concatenate([o.cache_features[:n][keep], [0]]).astype(np.uint32)
    data = np.concatenate([o.cache_data[:n][keep], np.zeros(1, scenes.IMPULSE)])
    order = np.lexsort((feats, tags))
    m = len(tags)
    o.cache_tags[:m] = tags[order]; o.cache_features[:m] = feats[order]; o.cache_data[:m] = data[order]; o.cache.count = m
    g = _sim(o.export_state(), o)   # uploads the bodies at the synced state
    g.cache_tags[:m] = o.cache_tags[:m]; g.cache_features[:m] = o.cache_features[:m]; g.cache_data[:m] = o.cache_data[:m]; g.cache.count = m
    g.upload_cache()
    rec = _recorder(o)
    first = rec.step()
    g.step_staged()
    _same(g.contact_events()[0], first, "first step after the upload")
    assert int(fake) in set(int(t) for t in first["tags"][first["kind"] == scenes.CONTACT_END])
    assert (first["kind"] == scenes.CONTACT_BEGIN).sum() >= len(keys[::3]) // 2
    for i in range(3):
        want = rec.step(); g.step_staged()
        _same(g.contact_events()[0], want, "step %d" % i)


def test_more_than_50k_contacts_from_an_emptied_cache():
    """Every pair of a settled wall begins again after its cache is emptied: the flags and the scatter span hundreds of scan tiles."""
    s = scenes.brick_wall(10000, iterations=8)
    o = _oracle(s)
    g = nudge_b200.Sim(s, contact_capacity=o.cap)
    for _ in range(60):
        g.step()
    assert g.counts().overflow == 0 and g.counts().contacts >= 50000
    sync_oracle_from_gpu(o, g)
    o.cache.count = 0; g.cache.count = 0
    g.upload_cache()
    g.enable_contact_events(1 << 17)
    rec = _recorder(o)
    for i in range(2):
        want = rec.step(); g.step_staged()
        _same(g.contact_events()[0], want, "step %d" % i)
        if i == 0:
            assert len(want) > 5000 and (want["kind"] == scenes.CONTACT_BEGIN).all()


def test_sharded_step_refuses_a_context_with_events():
    s = _falling()
    b = nudge_b200.Sim(s, stream=_stream())
    b.shard_create(0, 1, None, 1, 1)
    b.enable_contact_events(64)
    with pytest.raises(nudge_b200.NudgeError, match=r"\(-3\)"):
        b.shard_step("peer")
    b.enable_contact_events(0)
    b.shard_step("peer")
