"""The numpy restatement of nb_overlap (oracle/overlap_ref.py) on the CPU: analytic cases of the four tests (sphere-sphere exactly tangent,
sphere-box against a face, an edge and a corner, a point query on a face, box-box face to face, a rotated pair that only an edge-edge cross
axis separates, parallel boxes with zero cross axes, a box query containing colliders), degenerate queries, masks, ignore_body, sensors,
the result's order and offsets, and the nb_overlap_query / nb_overlap_hit layouts of nudge_b200/abi.py against the header."""
import os
import subprocess
import numpy as np
from nudge_b200 import abi, scenes
from oracle import overlap_ref
from tests.test_raycast_ref import _scene, UNIT, S45, ROOT

NAN, INF = float("nan"), float("inf")
ID = (0.0, 0.0, 0.0, 1.0)


def _q(shape, c, r=0.0, rot=ID, h=(0.0, 0.0, 0.0), mask=0xffffffff, ignore=abi.RAY_NO_HIT):
    q = np.zeros(1, abi.OVERLAP_QUERY)
    q["shape"], q["center"], q["radius"], q["rotation"], q["half_extents"], q["mask"], q["ignore_body"] = shape, c, r, rot, h, mask, ignore
    return q


def sphere(c, r, **kw):
    return _q(abi.OVERLAP_SPHERE, c, r=r, **kw)


def box(c, h, rot=ID, **kw):
    return _q(abi.OVERLAP_BOX, c, rot=rot, h=h, **kw)


def _hits(scene, q, flags=0):
    off, hits = overlap_ref.query(scene, q, flags)
    assert off[0] == 0 and off[-1] == len(hits)
    return list(hits["collider"])


def below(x):
    return float(np.nextafter(np.float32(x), np.float32(-INF)))


def above(x):
    return float(np.nextafter(np.float32(x), np.float32(INF)))


def test_sphere_sphere_exactly_tangent():
    s = _scene(spheres=[((3.0, 0.0, 0.0), 2.0)])
    assert _hits(s, sphere((0.0, 0.0, 0.0), 1.0)) == [0]            # 9 <= 3 * 3: touching counts
    assert _hits(s, sphere((below(0.0), 0.0, 0.0), 1.0)) == [0]      # d.x rounds to 3 again
    assert _hits(_scene(spheres=[((above(3.0), 0.0, 0.0), 2.0)]), sphere((0.0, 0.0, 0.0), 1.0)) == []   # 9.000002 > 9
    assert _hits(s, sphere((0.0, 4.0, 0.0), 3.0)) == [0]            # d = (-3, 4, 0): 25 <= 5 * 5
    assert _hits(s, sphere((0.0, above(4.0), 0.0), 3.0)) == []


def test_sphere_against_a_box_face_edge_and_corner():
    s = _scene([UNIT])
    assert _hits(s, sphere((2.0, 0.0, 0.0), 1.0)) == [0]            # face: g = (1, 0, 0)
    assert _hits(s, sphere((2.0, 0.0, 0.0), below(1.0))) == []
    assert _hits(s, sphere((4.0, 5.0, 0.0), 5.0)) == [0]            # edge: g = (3, 4, 0)
    assert _hits(s, sphere((4.0, 5.0, 0.0), below(5.0))) == []
    assert _hits(s, sphere((-3.0, 4.0, -7.0), 7.0)) == [0]          # corner: g = (-2, 3, -6)
    assert _hits(s, sphere((-3.0, 4.0, -7.0), below(7.0))) == []
    assert _hits(s, sphere((0.5, 0.25, -0.5), 0.0)) == [0]          # a point inside
    assert _hits(s, sphere((1.0, 0.5, 0.25), 0.0)) == [0]           # a point on a face: r = 0
    assert _hits(s, sphere((above(1.0), 0.5, 0.25), 0.0)) == []


def test_rotated_box_collider_and_box_query_against_a_sphere():
    s = _scene([((0.0, 0.0, 0.0), (2.0, 1.0, 1.0), (0.0, 0.0, S45, S45))])   # the long axis turned onto y
    assert _hits(s, sphere((0.0, 2.5, 0.0), 0.5)) == [0]
    assert _hits(s, sphere((2.5, 0.0, 0.0), 0.5)) == []
    sp = _scene(spheres=[((0.0, 3.0, 0.0), 1.0)])
    assert _hits(sp, box((0.0, 0.0, 0.0), (2.0, 1.0, 1.0), (0.0, 0.0, S45, S45))) == [0]   # reaches y = 2, the sphere y = 2
    assert _hits(sp, box((0.0, 0.0, 0.0), (2.0, 1.0, 1.0))) == []
    assert _hits(sp, box((0.0, 0.0, 0.0), (1.0, 2.0, 1.0))) == [0]   # touching


def test_box_box_face_to_face_at_integer_coordinates():
    s = _scene([UNIT])
    assert _hits(s, box((2.0, 0.0, 0.0), (1.0, 1.0, 1.0))) == [0]   # |t.x| = 2 > 1 + 1 is false: touching overlaps
    assert _hits(s, box((0.0, -3.0, 0.0), (1.0, 2.0, 1.0))) == [0]
    assert _hits(s, box((2.0, 2.0, 2.0), (1.0, 1.0, 1.0))) == [0]   # corner to corner
    assert _hits(s, box((3.0, 0.0, 0.0), (1.0, 1.0, 1.0))) == []
    assert _hits(s, box((above(2.0), 0.0, 0.0), (1.0, 1.0, 1.0))) == []


def _face_axes_separate(c, rot, H, p, q, h):
    """Whether one of the six face axes of the header's box-box test separates (float64 is enough here)."""
    axes = lambda r: [np.array(overlap_ref.qrot(tuple(np.float64(x) for x in r), tuple(np.eye(3)[k]))) for k in range(3)]
    u, v = axes(rot), axes(q)
    t = np.subtract(p, c)
    for L in list(u) + list(v):
        if abs(t @ L) > sum(abs(H[k] * (u[k] @ L)) for k in range(3)) + sum(abs(h[k] * (v[k] @ L)) for k in range(3)):
            return True
    return False


def test_a_pair_only_an_edge_cross_axis_separates():
    """The query turned 45 degrees about z has an edge along z at y = sqrt(2); the collider turned 45 degrees about x has one along x at
    y = 3 - sqrt(2).  Only cross(u_z, v_x) = y separates them; every face axis overlaps up to y = 3.83."""
    s8, c8 = float(np.sin(np.pi / 8)), float(np.cos(np.pi / 8))
    rz, rx = (0.0, 0.0, s8, c8), (s8, 0.0, 0.0, c8)
    s = _scene([((0.0, 3.0, 0.0), (1.0, 1.0, 1.0), rx)])
    assert not _face_axes_separate((0.0, 0.0, 0.0), rz, (1, 1, 1), (0.0, 3.0, 0.0), rx, (1, 1, 1))
    assert _hits(s, box((0.0, 0.0, 0.0), (1.0, 1.0, 1.0), rz)) == []
    assert _hits(s, box((0.0, 0.5, 0.0), (1.0, 1.0, 1.0), rz)) == [0]   # the edges cross: y gap 2.5 < 2 sqrt(2)


def test_parallel_boxes_with_zero_cross_axes():
    f = np.float32
    e = [tuple(f(x) for x in row) for row in np.eye(3)]
    u = [overlap_ref.qrot(tuple(f(x) for x in ID), r) for r in e]
    assert all(overlap_ref.dot(overlap_ref.cross(u[k], u[k]), overlap_ref.cross(u[k], u[k])) == 0 for k in range(3))
    s = _scene([((5.0, 5.0, 5.0), (1.0, 2.0, 3.0), ID)])
    assert _hits(s, box((5.0, 5.0, 9.0), (1.0, 1.0, 1.0))) == [0]    # touching on z: the zero axes cannot separate
    assert _hits(s, box((7.5, 5.0, 5.0), (1.0, 1.0, 1.0))) == []     # separated on x
    assert _hits(s, box((5.0, 5.0, 5.0), (0.5, 0.5, 0.5))) == [0]    # contained


def test_a_box_query_that_contains_colliders():
    s = _scene([((1.0, 2.0, 3.0), (0.5, 0.5, 0.5), (0.0, S45, 0.0, S45))], [((-2.0, 1.0, 0.0), 0.5), ((30.0, 0.0, 0.0), 0.5)])
    off, hits = overlap_ref.query(s, np.concatenate([box((0.0, 0.0, 0.0), (10.0, 10.0, 10.0), (0.0, 0.0, S45, S45)),
                                                     sphere((0.0, 0.0, 0.0), 100.0), sphere((100.0, 0.0, 0.0), 1.0)]))
    assert list(off) == [0, 2, 5, 5]
    assert list(hits["query"]) == [0, 0, 1, 1, 1] and list(hits["collider"]) == [0, 1, 0, 1, 2]
    assert list(hits["body"]) == [1, 2, 1, 2, 3] and list(hits["tag"]) == [100, 101, 100, 101, 102]


def test_degenerate_queries_hit_nothing():
    s = _scene([UNIT], [((0.0, 0.0, 0.0), 1.0)])
    bad = [_q(2, (0.0, 0.0, 0.0), r=1.0), sphere((NAN, 0.0, 0.0), 1.0), sphere((0.0, 0.0, 0.0), INF), sphere((0.0, 0.0, 0.0), -1.0),
           sphere((0.0, 0.0, 0.0), NAN), box((0.0, INF, 0.0), (1.0, 1.0, 1.0)), box((0.0, 0.0, 0.0), (1.0, -1.0, 1.0)),
           box((0.0, 0.0, 0.0), (1.0, 1.0, NAN)), box((0.0, 0.0, 0.0), (1.0, 1.0, 1.0), (0.0, 0.0, 0.0, 0.0)),
           box((0.0, 0.0, 0.0), (1.0, 1.0, 1.0), (1e-30, 0.0, 0.0, 1e-30)), box((0.0, 0.0, 0.0), (1.0, 1.0, 1.0), (0.0, NAN, 0.0, 1.0))]
    off, hits = overlap_ref.query(s, np.concatenate(bad))
    assert len(hits) == 0 and (off == 0).all()
    # fields a shape does not read are not read: a sphere's rotation and half extents, a box's radius
    ok = [sphere((0.0, 0.0, 0.0), 0.5, rot=(NAN, 0.0, 0.0, 0.0), h=(-1.0, INF, NAN)), box((0.0, 0.0, 0.0), (0.5, 0.5, 0.5), rot=(0.0, 0.0, 0.0, 2.0))]
    ok[1]["radius"] = -NAN
    off, hits = overlap_ref.query(s, np.concatenate(ok))
    assert list(off) == [0, 2, 4]   # a rotation used as given: (0, 0, 0, 2) is not normalised and still valid


def test_masks_ignore_body_and_sensors():
    filt = np.zeros(3, scenes.FILTER); filt["category"] = (0x0002, 0x0004, 0x0002)
    s = _scene([UNIT, ((3.0, 0.0, 0.0), (1.0, 1.0, 1.0), ID)], [((0.0, 3.0, 0.0), 1.0)], filters=filt, sensors=np.array([1, 0, 0], np.uint8))
    q = lambda **kw: sphere((0.0, 0.0, 0.0), 5.0, **kw)
    assert _hits(s, q()) == [1, 2]                                   # the sensor is skipped by default
    assert _hits(s, q(), abi.OVERLAP_SENSORS) == [0, 1, 2]
    assert _hits(s, q(mask=0x0002), abi.OVERLAP_SENSORS) == [0, 2]
    assert _hits(s, q(mask=0x0001), abi.OVERLAP_SENSORS) == []
    assert _hits(s, q(ignore=2)) == [2]
    assert _hits(s, q(ignore=3), abi.OVERLAP_SENSORS) == [0, 1]


def test_overlap_layouts_match_the_header(tmp_path):
    for dt, name in ((abi.OVERLAP_QUERY, "nb_overlap_query"), (abi.OVERLAP_HIT, "nb_overlap_hit")):
        src = tmp_path / "layout.c"
        src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "nudge_b200.h"\nint main(void) {\n' +
                       "".join('printf("%%zu\\n", offsetof(%s, %s));\n' % (name, k) for k in dt.names) +
                       'printf("%%zu\\n", sizeof(%s)); printf("%%d %%d %%d\\n", (int)NB_OVERLAP_SPHERE, (int)NB_OVERLAP_BOX, (int)NB_OVERLAP_SENSORS);'
                       ' return 0; }\n' % name)
        exe = tmp_path / "layout"
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), "-o", str(exe), str(src)])
        out = [int(x) for x in subprocess.check_output([str(exe)]).split()]
        assert out[:len(dt.names)] == [dt.fields[k][1] for k in dt.names]
        assert out[len(dt.names):] == [dt.itemsize, abi.OVERLAP_SPHERE, abi.OVERLAP_BOX, abi.OVERLAP_SENSORS]
    assert abi.OVERLAP_QUERY.itemsize == 64 and abi.OVERLAP_HIT.itemsize == 16
