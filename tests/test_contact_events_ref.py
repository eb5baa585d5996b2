"""The contact-event restatement (oracle/events_ref.py) on hand-built cases and over a CPU-oracle run with sleeping islands, and the
nb_contact_event layout against the header.  CPU only."""
import os, shutil, subprocess
import numpy as np
import pytest
from nudge_b200 import scenes as S
from oracle import events_ref as ER
from oracle.pyoracle import OracleSim

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BEGIN, END = S.CONTACT_BEGIN, S.CONTACT_END


def key(a, b):
    return a | (b << 32)


def contacts(rows):
    """rows: (tag, feature, penetration, body_a, body_b) -> a contacts_view()-like dict; position = (i, 2i, 3i), normal = (0, 1, i)."""
    n = len(rows)
    d = dict(tags=np.zeros(n, np.uint64), features=np.zeros(n, np.uint32), data=np.zeros(n, S.CONTACT), bodies=np.zeros(n, S.PAIR32))
    for i, (t, f, pen, a, b) in enumerate(rows):
        d["tags"][i] = t; d["features"][i] = f
        d["data"][i]["penetration"] = pen; d["data"][i]["position"] = (i, 2 * i, 3 * i); d["data"][i]["normal"] = (0, 1, i)
        d["bodies"][i] = (a, b)
    return d


def run(old, rows, culled=(), impulses=None, step=0):
    c = contacts(rows)
    imp = np.zeros((len(rows), 3), np.float32) if impulses is None else np.asarray(impulses, np.float32)
    return ER.events(np.array(old, np.uint64), c, imp, np.array(culled, np.uint64), step)


def test_begin_end_and_persist_in_key_order():
    k1, k2, k3, k4 = key(5, 1), key(3, 2), key(7, 2), key(9, 0)
    ev = run([k4, k1, k2, k2], [(k3, 1, 0.1, 3, 4), (k2, 0, 0.2, 1, 2)], step=7)
    # k4 and k1 ended (ascending key order), k3 began, k2 persisted
    assert list(ev["kind"]) == [END, END, BEGIN]
    assert list(ev["tags"]) == sorted([k4, k1]) + [k3]
    assert (ev["step"] == 7).all()
    end = ev[ev["kind"] == END]
    for f in ("body_a", "body_b", "contacts", "penetration", "position", "normal", "impulse"):
        assert not np.any(end[f]), f
    b = ev[2]
    assert b["contacts"] == 1 and (b["body_a"], b["body_b"]) == (3, 4) and np.float32(b["penetration"]) == np.float32(0.1)


def test_sleeping_pair_never_ends():
    k = key(4, 1)
    assert len(run([k, k], [], culled=[k, k])) == 0


def test_waking_pair_ends_when_gone_and_does_not_begin_again_when_touching():
    k = key(4, 1)
    ev = run([k], [])                        # its island woke (not culled) and the pair is gone
    assert list(ev["kind"]) == [END] and ev[0]["tags"] == k
    assert len(run([k], [(k, 0, 0.1, 1, 2)])) == 0   # woke still touching: in old and in cur


def test_deepest_contact_ties_keep_the_first_and_nan_never_wins():
    k = key(6, 2)
    # input order differs from (tag, feature) order: feature 0 comes first in the walk
    ev = run([], [(k, 3, 0.5, 9, 9), (k, 0, 0.5, 1, 2), (k, 1, 0.25, 5, 5)])
    assert ev[0]["contacts"] == 3 and (ev[0]["body_a"], ev[0]["body_b"]) == (1, 2)
    assert tuple(ev[0]["position"]) == (1, 2, 3)
    ev = run([], [(k, 0, np.nan, 1, 2), (k, 1, 0.5, 5, 5)])
    assert np.isnan(ev[0]["penetration"]) and ev[0]["body_a"] == 1
    ev = run([], [(k, 0, 0.5, 1, 2), (k, 1, np.nan, 5, 5), (k, 2, 0.75, 7, 7)])
    assert ev[0]["penetration"] == np.float32(0.75) and ev[0]["body_a"] == 7


def test_impulse_is_the_sequential_fp32_sum_in_tag_order():
    k = key(6, 2)
    vals = [1e8, 1.0, -1e8, 1.0]
    rows = [(k, f, 0.1, 1, 2) for f in range(4)]
    imp = np.zeros((4, 3), np.float32); imp[:, 1] = vals
    ev = run([], rows[::-1], impulses=imp[::-1])   # reversed input: the walk still goes by feature
    pairwise = np.float32(np.float32(vals[0] + vals[1]) + np.float32(vals[2] + vals[3]))
    assert ev[0]["impulse"][1] == np.float32(1.0) and pairwise != np.float32(1.0)


def test_touching_sets_follow_the_events_over_an_oracle_run_with_sleeping_islands():
    s = S.demo_scene(120, 120, iterations=4, spread=6.0, height=6.0, seed=11)
    o = OracleSim(s)
    rec = ER.OracleEvents(o)
    prev = ER.touching(o.cache_view())
    kinds = {BEGIN: 0, END: 0}
    slept = 0
    for i in range(60):
        if i == 40:   # put most islands to sleep (the idle counter saturates at 0xff)
            sleepy = np.random.default_rng(5).random(s.n_bodies) < 0.8
            o.idle[sleepy] = 0xff
            o.momentum["velocity"][sleepy] = 0; o.momentum["angular_velocity"][sleepy] = 0
        ev = rec.step()
        assert (ev["step"] == i).all()
        ends = set(int(t) for t in ev["tags"][ev["kind"] == END])
        begins = set(int(t) for t in ev["tags"][ev["kind"] == BEGIN])
        cur = ER.touching(o.cache_view())
        assert cur == (prev - ends) | begins and not (ends & begins)
        prev = cur
        kinds[BEGIN] += len(begins); kinds[END] += len(ends)
        slept = max(slept, o.contacts.sleeping_count)
    assert kinds[BEGIN] > 0 and kinds[END] > 0 and slept > 0


def test_event_struct_layout_matches_the_header(tmp_path):
    cxx = shutil.which("g++") or shutil.which("cc")
    if not cxx:
        pytest.skip("no host C compiler")
    src = tmp_path / "layout.cpp"
    src.write_text('#include "nudge_b200.h"\n#include <stdio.h>\n#include <stddef.h>\nint main() { printf("%zu %zu %zu %zu %zu %zu %zu %zu %zu %zu %zu %zu\\n", sizeof(nb_contact_event), '
                   + ", ".join("offsetof(nb_contact_event, %s)" % f for f in ("tags", "kind", "step", "body_a", "body_b", "contacts", "penetration", "position", "normal", "impulse", "reserved"))
                   + "); return NB_CONTACT_BEGIN == 1 && NB_CONTACT_END == 2 ? 0 : 1; }\n")
    exe = tmp_path / "layout"
    subprocess.check_call([cxx, "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    got = [int(x) for x in subprocess.check_output([str(exe)]).split()]
    names = ("tags", "kind", "step", "body_a", "body_b", "contacts", "penetration", "position", "normal", "impulse", "reserved")
    assert got == [S.CONTACT_EVENT.itemsize] + [S.CONTACT_EVENT.fields[n][1] for n in names]
