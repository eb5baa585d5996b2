"""The contact impulse restatement (tests/contact_impulse_ref.py) on hand-built contact sets: the sign and the lever arm of one contact, a
contact whose two sides name the same body, body 0 summing several pairs, duplicate tags merging into one pair row, the threshold, the
capacity and the count, out-of-range indices in host and device semantics, and the struct layouts against the header.  CPU only."""
import os
import subprocess
import numpy as np
import pytest
from nudge_b200 import abi, scenes
from tests.contact_impulse_ref import REMOVED, body_report, body_report_loop, pair_report, pair_rows

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
f32 = np.float32


@pytest.mark.parametrize("dt,name,size", [(abi.BODY_CONTACT_IMPULSE, "nb_body_contact_impulse", 32),
                                          (abi.CONTACT_PAIR_IMPULSE, "nb_contact_pair_impulse", 48)])
def test_layouts_match_the_header(tmp_path, dt, name, size):
    src = tmp_path / "layout.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "nudge_b200.h"\nint main(void) {\n' +
                   "".join('printf("%%zu\\n", offsetof(%s, %s));\n' % (name, k) for k in dt.names) +
                   'printf("%%zu\\n", sizeof(%s)); return 0; }\n' % name)
    exe = tmp_path / "layout"
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), "-o", str(exe), str(src)])
    out = [int(x) for x in subprocess.check_output([str(exe)]).split()]
    assert out == [dt.fields[k][1] for k in dt.names] + [size]


def _set(rows):
    """rows: (a, b, tags, feature, position, normal, penetration, J)."""
    n = len(rows)
    data = np.zeros(n, scenes.CONTACT); bodies = np.zeros(n, scenes.PAIR32); tags = np.zeros(n, np.uint64); J = np.zeros((n, 3), f32)
    for i, (a, b, t, _, p, nrm, pen, j) in enumerate(rows):
        bodies[i] = (a, b); tags[i] = t; data["position"][i] = p; data["normal"][i] = nrm; data["penetration"][i] = pen; J[i] = j
    feat = np.array([r[3] for r in rows], np.uint64)
    sorted_idx = np.lexsort((feat, tags)).astype(np.uint32)   # (tag, feature) order
    return data, bodies, tags, J, sorted_idx


def test_sign_and_lever_arm_of_one_contact():
    pos = np.array([(0, 0, 0), (1, 2, 3), (0, 5, 0)], f32)
    data, bodies, tags, J, srt = _set([(1, 2, 1 | 2 << 32, 0, (1.5, 2.0, 3.0), (0, 1, 0), 0.01, (0.0, 3.0, 0.5))])
    out = body_report(data, bodies, J, pos, 3)
    r_a = np.array((0.5, 0.0, 0.0), f32); r_b = np.array((1.5, -3.0, 3.0), f32)
    j = J[0]
    assert (out["impulse"][1] == -j).all() and (out["impulse"][2] == j).all()
    assert (out["angular_impulse"][1] == -np.cross(r_a, j)).all() and (out["angular_impulse"][2] == np.cross(r_b, j)).all()
    assert list(out["contacts"]) == [0, 1, 1] and list(out["body"]) == [0, 1, 2]
    assert (out["impulse"][0] == 0).all() and (out["angular_impulse"][0] == 0).all()


def test_a_contact_on_one_body_counts_both_sides():
    pos = np.array([(0, 0, 0), (0, 1, 0)], f32)
    data, bodies, tags, J, srt = _set([(1, 1, 7 | 7 << 32, 0, (0.5, 1.0, 0.0), (0, 1, 0), 0.0, (0.25, 1.0, -2.0))])
    out = body_report(data, bodies, J, pos, 2)
    assert out["contacts"][1] == 2
    # -J then +J: exactly zero for these values, and the torque cancels the same way (same lever arm)
    assert (out["impulse"][1] == (f32(0) - J[0]) + J[0]).all()
    assert (out["angular_impulse"][1] == 0).all()


def _random_set(rng, n_bodies=12, n=300, duplicate_tags=False):
    a = rng.integers(0, n_bodies, n); b = rng.integers(0, n_bodies, n)
    a[: n // 5] = 0   # body 0 in many pairs
    tagpool = rng.integers(1, 40 if duplicate_tags else 1 << 30, (n, 2))
    rows = []
    for i in range(n):
        t = int(min(tagpool[i])) | int(max(tagpool[i])) << 32
        rows.append((a[i], b[i], t, int(rng.integers(0, 8)), rng.normal(0, 3, 3), rng.normal(0, 1, 3), rng.uniform(-0.01, 0.05),
                     rng.normal(0, 2, 3)))
    return _set(rows), rng.normal(0, 3, (n_bodies, 3)).astype(f32)


def test_body_0_sums_several_pairs_in_contact_order():
    rng = np.random.default_rng(3)
    (data, bodies, tags, J, srt), pos = _random_set(rng)
    out = body_report(data, bodies, J, pos, 12)
    for b in range(12):
        acc, tq, k = body_report_loop(data, bodies, J, pos, b)
        assert out["impulse"][b].tobytes() == acc.tobytes() and out["angular_impulse"][b].tobytes() == tq.tobytes() and out["contacts"][b] == k
    assert out["contacts"][0] >= 60
    # the order matters: the same sides summed in reverse give other bits for at least one body
    rev = body_report(data[::-1].copy(), bodies[::-1].copy(), J[::-1].copy(), pos, 12)
    assert (rev["impulse"] != out["impulse"]).any()


def test_duplicate_tags_merge_into_one_pair_row():
    n = (0, 1, 0)
    data, bodies, tags, J, srt = _set([(1, 2, 5 | 9 << 32, 3, (0, 0, 0), n, 0.01, (0, 1, 0)),
                                       (3, 4, 5 | 9 << 32, 1, (1, 0, 0), n, 0.03, (0, 2, 0)),   # another collider pair, the same key
                                       (1, 2, 5 | 9 << 32, 2, (2, 0, 0), n, 0.03, (0.5, 4, 0)),  # a tie: the earlier contact stays deepest
                                       (0, 1, 2 | 5 << 32, 0, (3, 0, 0), n, 0.02, (0, 8, 0))])
    rows = pair_rows(data, bodies, tags, J, srt)
    assert list(rows["tags"]) == [2 | 5 << 32, 5 | 9 << 32]
    r = rows[1]
    assert r["contacts"] == 3 and r["body_a"] == 3 and r["body_b"] == 4 and r["penetration"] == f32(0.03)
    # (tag, feature) order: features 1, 2, 3 -> contacts 1, 2, 0
    want = (f32(0) + J[1]) + J[2]; want = want + J[0]
    assert r["impulse"].tobytes() == want.astype(f32).tobytes()
    assert r["normal_impulse"] == ((f32(0) + f32(2)) + f32(4)) + f32(1)
    assert list(r["reserved"]) == [0, 0]


def test_a_nan_penetration_never_wins():
    n = (0, 1, 0)
    data, bodies, tags, J, srt = _set([(1, 2, 1 | 2 << 32, 0, (0, 0, 0), n, np.nan, (0, 1, 0)),
                                       (3, 4, 1 | 2 << 32, 1, (0, 0, 0), n, 0.5, (0, 1, 0)),
                                       (5, 6, 1 | 2 << 32, 2, (0, 0, 0), n, np.nan, (0, 1, 0))])
    r = pair_rows(data, bodies, tags, J, srt)[0]
    # the first contact's NaN depth is never beaten: "p > NaN" is false
    assert r["body_a"] == 1 and np.isnan(r["penetration"])


def test_threshold_capacity_and_count():
    rng = np.random.default_rng(5)
    (data, bodies, tags, J, srt), pos = _random_set(rng, n=200)
    rows = pair_rows(data, bodies, tags, J, srt)
    assert (np.diff(rows["tags"].astype(np.float64)) > 0).all()
    every, n_every = pair_report(data, bodies, tags, J, srt, -np.inf)
    assert n_every == len(rows) and every.tobytes() == rows.tobytes()
    zero, n_zero = pair_report(data, bodies, tags, J, srt, 0.0)
    assert n_zero == int((rows["normal_impulse"] >= 0).sum()) and 0 < n_zero < len(rows)
    cut = np.sort(rows["normal_impulse"])[len(rows) // 2]
    kept, n_kept = pair_report(data, bodies, tags, J, srt, cut)
    assert n_kept == int((rows["normal_impulse"] >= cut).sum()) and (kept["normal_impulse"] >= cut).all()
    assert kept.tobytes() == rows[rows["normal_impulse"] >= cut].tobytes()
    short, n_short = pair_report(data, bodies, tags, J, srt, -np.inf, capacity=7)
    assert n_short == len(rows) and short.tobytes() == rows[:7].tobytes()
    none, n_none = pair_report(data, bodies, tags, J, srt, -np.inf, capacity=0)
    assert len(none) == 0 and n_none == len(rows)
    with pytest.raises(ValueError):
        pair_report(data, bodies, tags, J, srt, np.nan)


def test_out_of_range_indices_host_and_device():
    rng = np.random.default_rng(9)
    (data, bodies, tags, J, srt), pos = _random_set(rng)
    idx = np.array([3, 12, 0, REMOVED, 11, 3], np.uint32)
    with pytest.raises(ValueError):
        body_report(data, bodies, J, pos, 12, idx)
    out = body_report(data, bodies, J, pos, 12, idx, device=True)
    full = body_report(data, bodies, J, pos, 12)
    for i, b in enumerate(idx):
        if b < 12:
            assert out[i].tobytes() == full[b].tobytes()
        else:
            assert out["body"][i] == REMOVED and out["contacts"][i] == 0
            assert (out["impulse"][i] == 0).all() and (out["angular_impulse"][i] == 0).all()
