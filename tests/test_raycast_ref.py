"""The numpy restatement of nb_raycast (oracle/raycast_ref.py) on the CPU: analytic cases of the box and sphere tests (axis-aligned and
rotated boxes, spheres, origins inside, rays parallel to a slab inside and outside it, a grazing edge, max_t stopping short, ties,
degenerate rays, masks, ignore_body and sensors), and the nb_ray / nb_ray_hit layouts of nudge_b200/abi.py against the header."""
import os
import subprocess
import numpy as np
from nudge_b200 import abi, scenes
from oracle import raycast_ref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
S45 = float(np.sin(np.pi / 4))


def _scene(boxes=(), spheres=(), filters=None, sensors=None):
    """boxes: (position, half extents, rotation, body); spheres: (position, radius, body).  Every collider sits at its body's origin; body
    k + 1 carries the position and rotation."""
    items = list(boxes) + list(spheres)
    body = np.zeros(len(items) + 1, scenes.TRANSFORM); body["rotation"][:, 3] = 1.0
    bx = np.zeros(len(boxes), scenes.TRANSFORM); sx = np.zeros(len(spheres), scenes.TRANSFORM)
    bx["rotation"][:, 3] = 1.0; sx["rotation"][:, 3] = 1.0
    bd = np.zeros(len(boxes), scenes.BOX); sd = np.zeros(len(spheres), scenes.SPHERE)
    for k, (p, h, q, *b) in enumerate(boxes):
        body["position"][k + 1], body["rotation"][k + 1], bd["size"][k] = p, q, h
        bx["body"][k] = b[0] if b else k + 1
    for k, (p, r, *b) in enumerate(spheres):
        body["position"][len(boxes) + k + 1], sd["radius"][k] = p, r
        sx["body"][k] = b[0] if b else len(boxes) + k + 1
    tags = np.arange(len(items), dtype=np.uint32) + 100
    return raycast_ref.Scene(body, bx, bd, tags[:len(boxes)], sx, sd, tags[len(boxes):], filters, sensors)


def _ray(o, d, max_t=100.0, mask=0xffffffff, ignore=abi.RAY_NO_HIT):
    r = np.zeros(1, abi.RAY)
    r["origin"], r["direction"], r["max_t"], r["mask"], r["ignore_body"] = o, d, max_t, mask, ignore
    return r


def _cast(scene, *args, flags=0, **kw):
    return raycast_ref.cast(scene, _ray(*args, **kw), flags)[0]


UNIT = ((0.0, 0.0, 0.0), (1.0, 1.0, 1.0), (0.0, 0.0, 0.0, 1.0))


def _is_miss(h):
    return h["collider"] == h["body"] == h["tag"] == abi.RAY_NO_HIT and h.tobytes()[:28] == bytes(28) and h.tobytes()[40:] == bytes(8)


def test_axis_aligned_box():
    s = _scene([UNIT])
    h = _cast(s, (-5.0, 0.0, 0.0), (1.0, 0.0, 0.0))
    assert h["t"] == 4.0 and tuple(h["position"]) == (-1.0, 0.0, 0.0) and tuple(h["normal"]) == (-1.0, 0.0, 0.0)
    assert (h["collider"], h["body"], h["tag"]) == (0, 1, 100)
    h = _cast(s, (0.0, 0.0, 5.0), (0.0, 0.0, -2.0))   # direction not unit: t in units of its length
    assert h["t"] == 2.0 and tuple(h["normal"]) == (0.0, 0.0, 1.0)
    assert _is_miss(_cast(s, (-5.0, 0.0, 0.0), (-1.0, 0.0, 0.0)))   # pointing away


def test_rotated_box():
    s = _scene([((0.0, 0.0, 0.0), (2.0, 1.0, 1.0), (0.0, 0.0, S45, S45))])   # the long axis turned onto y
    h = _cast(s, (0.0, -5.0, 0.0), (0.0, 1.0, 0.0))
    assert abs(h["t"] - 3.0) < 1e-5 and np.allclose(h["normal"], (0.0, -1.0, 0.0), atol=1e-6)
    h = _cast(s, (-5.0, 0.0, 0.0), (1.0, 0.0, 0.0))
    assert abs(h["t"] - 4.0) < 1e-5 and np.allclose(h["normal"], (-1.0, 0.0, 0.0), atol=1e-6)


def test_sphere():
    s = _scene(spheres=[((0.0, 2.0, 0.0), 1.0)])
    h = _cast(s, (0.0, 7.0, 0.0), (0.0, -1.0, 0.0))
    assert h["t"] == 4.0 and tuple(h["position"]) == (0.0, 3.0, 0.0) and tuple(h["normal"]) == (0.0, 1.0, 0.0)
    assert _is_miss(_cast(s, (0.0, 7.0, 0.0), (0.0, 1.0, 0.0)))
    assert _is_miss(_cast(s, (1.5, 7.0, 0.0), (0.0, -1.0, 0.0)))


def test_origin_inside():
    s = _scene([UNIT], [((5.0, 0.0, 0.0), 1.0)])
    for o in ((0.2, 0.3, -0.1), (5.5, 0.0, 0.0)):
        h = _cast(s, o, (0.0, 1.0, 0.0))
        assert h["t"] == 0.0 and h["normal"].tobytes() == bytes(12) and tuple(h["position"]) == tuple(np.float32(o))
    assert _cast(s, (1.0, 0.0, 0.0), (1.0, 0.0, 0.0))["t"] == 0.0   # on the face counts as inside


def test_parallel_ray_inside_and_outside_a_slab():
    s = _scene([UNIT])
    assert _cast(s, (-5.0, 0.5, 0.0), (1.0, 0.0, 0.0))["t"] == 4.0
    assert _is_miss(_cast(s, (-5.0, 1.5, 0.0), (1.0, 0.0, 0.0)))
    assert _is_miss(_cast(s, (-5.0, 0.0, -1.01), (1.0, 0.0, 0.0)))


def test_grazing_edge():
    s = _scene([UNIT])
    h = _cast(s, (-5.0, 1.0, 1.0), (1.0, 0.0, 0.0))   # along the edge y = z = 1: closed slabs
    assert h["t"] == 4.0 and tuple(h["normal"]) == (-1.0, 0.0, 0.0)
    h = _cast(s, (-3.0, -3.0, 0.0), (1.0, 1.0, 0.0))  # through the edge x = y = -1: both axes enter at t = 2, x (the lower) wins
    assert h["t"] == 2.0 and tuple(h["normal"]) == (-1.0, 0.0, 0.0)


def test_max_t():
    s = _scene([UNIT], [((0.0, 0.0, 10.0), 1.0)])
    assert _is_miss(_cast(s, (-5.0, 0.0, 0.0), (1.0, 0.0, 0.0), max_t=3.99))
    assert _cast(s, (-5.0, 0.0, 0.0), (1.0, 0.0, 0.0), max_t=4.0)["t"] == 4.0
    assert _is_miss(_cast(s, (0.0, 0.0, 5.0), (0.0, 0.0, 1.0), max_t=3.5))
    assert _cast(s, (0.0, 0.0, 5.0), (0.0, 0.0, 1.0), max_t=4.0)["collider"] == 1


def test_ties_go_to_the_smaller_collider_index():
    s = _scene([UNIT, UNIT], [((0.0, 0.0, 0.0), 1.0)])
    assert _cast(s, (-5.0, 0.0, 0.0), (1.0, 0.0, 0.0))["collider"] == 0
    s = _scene([((0.0, 0.0, 0.0), (1.0, 1.0, 1.0), (0.0, 0.0, 0.0, 1.0), 2)], [((0.0, 0.0, 0.0), 1.0, 1)])
    h = _cast(s, (-5.0, 0.0, 0.0), (1.0, 0.0, 0.0))   # the sphere (index 1) ties with the box (index 0) at t = 4
    assert h["t"] == 4.0 and h["collider"] == 0
    assert _cast(s, (-5.0, 0.0, 0.0), (1.0, 0.0, 0.0), ignore=2)["collider"] == 1


def test_degenerate_rays():
    s = _scene([UNIT])
    nan, inf = float("nan"), float("inf")
    for o, d, mt in (((nan, 0, 0), (1, 0, 0), 10), ((-5, 0, 0), (inf, 0, 0), 10), ((-5, 0, 0), (0, 0, 0), 10), ((-5, 0, 0), (1, 0, 0), -1),
                     ((-5, 0, 0), (1, 0, 0), nan), ((-5, 0, 0), (1, 0, 0), inf), ((-5, 0, 0), (-0.0, 0.0, -0.0), 10)):
        assert _is_miss(_cast(s, o, d, max_t=mt)), (o, d, mt)


def test_mask_ignore_body_and_sensors():
    filt = np.zeros(2, scenes.FILTER); filt["category"] = (0x0002, 0x0004)
    s = _scene([UNIT, ((3.0, 0.0, 0.0), (1.0, 1.0, 1.0), (0.0, 0.0, 0.0, 1.0))], filters=filt, sensors=np.array([1, 0], np.uint8))
    o, d = (-5.0, 0.0, 0.0), (1.0, 0.0, 0.0)
    assert _cast(s, o, d)["collider"] == 1                           # the sensor is skipped by default
    assert _cast(s, o, d, flags=abi.RAY_SENSORS)["collider"] == 0
    assert _cast(s, o, d, mask=0x0004, flags=abi.RAY_SENSORS)["collider"] == 1
    assert _is_miss(_cast(s, o, d, mask=0x0001, flags=abi.RAY_SENSORS))
    assert _is_miss(_cast(s, o, d, ignore=2))


def test_ray_layouts_match_the_header(tmp_path):
    for dt, name in ((abi.RAY, "nb_ray"), (abi.RAY_HIT, "nb_ray_hit")):
        src = tmp_path / "layout.c"
        src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "nudge_b200.h"\nint main(void) {\n' +
                       "".join('printf("%%zu\\n", offsetof(%s, %s));\n' % (name, k) for k in dt.names) +
                       'printf("%%zu\\n", sizeof(%s)); printf("%%u\\n", (unsigned)NB_RAY_NO_HIT); printf("%%d\\n", (int)NB_RAY_SENSORS); return 0; }\n' % name)
        exe = tmp_path / "layout"
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), "-o", str(exe), str(src)])
        out = [int(x) for x in subprocess.check_output([str(exe)]).split()]
        assert out[:len(dt.names)] == [dt.fields[k][1] for k in dt.names]
        assert out[len(dt.names):] == [dt.itemsize, abi.RAY_NO_HIT, abi.RAY_SENSORS] and dt.itemsize == 48
