"""The body-state restatement (tests/body_state_ref.py) on the CPU: the row layout against the header, list order and duplicates, the wake
of a pose set (through the contact cache and through a connection, never a kinematic body or body 0), no partner wake for a velocity set,
and the gather.  CPU only."""
import os
import subprocess
import numpy as np
from nudge_b200 import abi, scenes
from tests.body_state_ref import REMOVED, get_states, set_states, valid
from tests.test_body_impulse_oracle import two_piles

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
POSE, VEL = abi.BODY_POSE, abi.BODY_VELOCITY


def test_body_state_layout_and_fields_match_the_header(tmp_path):
    dt, name = abi.BODY_STATE, "nb_body_state"
    src = tmp_path / "layout.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "nudge_b200.h"\nint main(void) {\n' +
                   "".join('printf("%%zu\\n", offsetof(%s, %s));\n' % (name, k) for k in dt.names) +
                   'printf("%%zu\\n", sizeof(%s)); printf("%%d\\n%%d\\n", (int)NB_BODY_POSE, (int)NB_BODY_VELOCITY); return 0; }\n' % name)
    exe = tmp_path / "layout"
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), "-o", str(exe), str(src)])
    out = [int(x) for x in subprocess.check_output([str(exe)]).split()]
    assert out == [dt.fields[k][1] for k in dt.names] + [64, abi.BODY_POSE, abi.BODY_VELOCITY]


def _live(seed=3):
    """Two stacks (two boxes and a sphere each) with random state; pile A = bodies 1, 2 and 5, pile B = 3, 4 and 6."""
    s, a, b = two_piles(height=2)
    rng = np.random.default_rng(seed)
    s.momentum["velocity"] = rng.normal(0.0, 1.0, (s.n_bodies, 3)); s.momentum["angular_velocity"] = rng.normal(0.0, 1.0, (s.n_bodies, 3))
    s.momentum["unused0"] = rng.normal(0.0, 1.0, s.n_bodies); s.momentum["unused1"] = rng.normal(0.0, 1.0, s.n_bodies)
    s.transforms["body"] = rng.integers(0, 1000, s.n_bodies)
    s.idle[:] = 0xff
    return s, a, b


def _tag(s, body):
    return int(s.box_tags[list(s.box_transforms["body"]).index(body)])


def _key(ta, tb):
    return np.uint64(ta) | (np.uint64(tb) << np.uint64(32))


def _rows(rng, bodies):
    r = np.zeros(len(bodies), abi.BODY_STATE)
    r["body"] = bodies
    for f, k in (("position", 3), ("rotation", 4), ("velocity", 3), ("angular_velocity", 3)):
        r[f] = rng.normal(0.0, 2.0, (len(bodies), k))
    r["idle_counter"] = 77; r["reserved"] = 5   # ignored by a set
    return r


def test_list_order_and_duplicates_last_entry_wins_per_field():
    s, a, b = _live()
    rng = np.random.default_rng(1)
    rows = _rows(rng, [2, 3, 2, 4, 2])
    for fields in (POSE, VEL, POSE | VEL):
        out, woken = set_states(s, rows, fields)
        for body, last in ((2, 4), (3, 1), (4, 3)):
            if fields & POSE:
                assert np.array_equal(out.transforms["position"][body], rows["position"][last])
                assert np.array_equal(out.transforms["rotation"][body], rows["rotation"][last])
            else:
                assert out.transforms[body].tobytes() == s.transforms[body].tobytes()
            if fields & VEL:
                assert np.array_equal(out.momentum["velocity"][body], rows["velocity"][last])
                assert np.array_equal(out.momentum["angular_velocity"][body], rows["angular_velocity"][last])
            else:
                assert out.momentum[body].tobytes() == s.momentum[body].tobytes()
            assert out.idle[body] == 0
        # the transform's body word and the momentum row's unused lanes stay; unlisted bodies stay
        assert np.array_equal(out.transforms["body"], s.transforms["body"])
        assert np.array_equal(out.momentum["unused0"], s.momentum["unused0"]) and np.array_equal(out.momentum["unused1"], s.momentum["unused1"])
        for body in (0, 1, 5, 6):
            assert out.transforms[body].tobytes() == s.transforms[body].tobytes() and out.momentum[body].tobytes() == s.momentum[body].tobytes()
    assert set_states(s, rows[::-1], VEL)[0].momentum[2].tobytes() == set_states(s, rows[:1], VEL)[0].momentum[2].tobytes()


def test_velocity_alone_wakes_no_partner():
    s, a, b = _live()
    s.connections = np.array([(a[0], a[1])], scenes.PAIR32)
    cache = [_key(_tag(s, a[0]), _tag(s, a[1])), _key(_tag(s, a[1]), 0)]
    out, woken = set_states(s, _rows(np.random.default_rng(2), [a[0]]), VEL, cache)
    assert np.nonzero(woken)[0].tolist() == [a[0]] and np.nonzero(out.idle == 0)[0].tolist() == [a[0]]


def test_a_pose_set_on_the_bottom_box_wakes_the_top_box_through_the_cache_and_through_a_connection():
    s, a, b = _live()
    bottom, top = int(a[0]), int(a[1])
    rows = _rows(np.random.default_rng(3), [bottom])
    ground = _tag(s, 0)
    # through the cache: the entry pairing the two boxes' tags (either order); the ground entry wakes nobody (body 0)
    for key in (_key(_tag(s, bottom), _tag(s, top)), _key(_tag(s, top), _tag(s, bottom))):
        out, woken = set_states(s, rows, POSE, [key, _key(ground, _tag(s, bottom))])
        assert np.nonzero(woken)[0].tolist() == [bottom, top] and out.idle[top] == 0 and out.idle[0] == s.idle[0]
    # an entry of pile B's boxes wakes nothing
    out, woken = set_states(s, rows, POSE, [_key(_tag(s, b[0]), _tag(s, b[1]))])
    assert np.nonzero(woken)[0].tolist() == [bottom]
    # through a connection, without a cache entry
    s.connections = np.array([(top, bottom), (b[0], b[1])], scenes.PAIR32)
    out, woken = set_states(s, rows, POSE, [])
    assert np.nonzero(woken)[0].tolist() == [bottom, top]
    # both sides moved: both listed, nobody else
    out, woken = set_states(s, _rows(np.random.default_rng(4), [bottom, top]), POSE | VEL, [_key(_tag(s, bottom), _tag(s, top))])
    assert np.nonzero(woken)[0].tolist() == [bottom, top]


def test_kinematic_bodies_are_written_and_never_woken():
    s, a, b = _live()
    k, partner = int(a[0]), int(a[1])
    s.kinematic = np.array([(partner, (0.0, 0.0, 0.0), (0.0, 0.0, 0.0), 0), (k, (0.0, 0.0, 0.0), (0.0, 0.0, 0.0), 0)], scenes.KINEMATIC)
    s.connections = np.array([(k, partner), (b[0], k)], scenes.PAIR32)
    rows = _rows(np.random.default_rng(5), [k])
    out, woken = set_states(s, rows, POSE | VEL, [_key(_tag(s, k), _tag(s, partner))], kinematic=[k, partner])
    assert np.array_equal(out.transforms["position"][k], rows["position"][0]) and np.array_equal(out.momentum["velocity"][k], rows["velocity"][0])
    assert out.idle[k] == 0xff and out.idle[partner] == 0xff   # written, not woken; the kinematic partner is not woken either
    assert np.nonzero(woken)[0].tolist() == [int(b[0])]        # the dynamic end of a connection to the moved kinematic body is


def test_validity_and_the_gather():
    s, a, b = _live()
    r = _rows(np.random.default_rng(6), [0, 1, s.n_bodies, 2, 3])
    r["velocity"][3, 1] = np.nan
    r["rotation"][4, 2] = np.inf
    assert valid(r, POSE, s.n_bodies).tolist() == [False, True, False, True, False]
    assert valid(r, VEL, s.n_bodies).tolist() == [False, True, False, False, True]
    g = get_states(s, [0, 5, s.n_bodies, 2])
    assert g["body"].tolist() == [0, 5, int(REMOVED), 2]
    assert g[2].tobytes() == np.array([(0,) * 3 + (REMOVED,) + (0,) * 4 + (0,) * 3 + (0,) + (0,) * 3 + (0,)], dtype="<f4,<f4,<f4,<u4,<f4,<f4,<f4,<f4,<f4,<f4,<f4,<u4,<f4,<f4,<f4,<u4").tobytes()
    assert np.array_equal(g["position"][1], s.transforms["position"][5]) and np.array_equal(g["angular_velocity"][3], s.momentum["angular_velocity"][2])
    assert g["idle_counter"][1] == 0xff and (g["reserved"] == 0).all()
    assert len(get_states(s)) == s.n_bodies and get_states(s)["body"].tolist() == list(range(s.n_bodies))
