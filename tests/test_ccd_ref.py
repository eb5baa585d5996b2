"""The numpy restatement of continuous collision (oracle/ccd_ref.py) on the CPU: analytic clamps (a sphere fired at a thin wall stops at its
face, also with the wall turned about the motion axis; a sphere target; the closer of two walls; ties to the smaller collider index; a
collider touched at the start skipped while a farther one still clamps), the threshold's strict >, +inf thresholds, bodies the step does
not advance, filters both ways, the connected skip, sensors and the body's own colliders; the tie to the two pinned restatements (with the
start skip off the hits are shapecast_ref's for the same sphere casts, and at radius 0 raycast_ref's rays); and the nb_ccd_body layout
against the header."""
import os
import subprocess
import numpy as np
from nudge_b200 import abi, scenes
from oracle import ccd_ref, overlap_ref, raycast_ref, shapecast_ref
from tests.test_raycast_ref import _scene, ROOT

INF = float("inf")
ID = (0.0, 0.0, 0.0, 1.0)
WALL = ((0.0, 0.0, 0.0), (0.1, 2.0, 2.0), ID)
f = np.float32


def _entry(body, radius, threshold=0.0, category=0xffff, mask=0xffff):
    e = np.zeros(1, abi.CCD_BODY)
    e["body"], e["radius"], e["motion_threshold"], e["category"], e["mask"] = body, radius, threshold, category, mask
    return e


def _one(scene, entry, p, d, **kw):
    t, c = ccd_ref.cast(scene, entry, np.array([p], f), np.array([d], f), **kw)
    return float(t[0]), int(c[0])


def test_a_sphere_fired_at_a_thin_wall_stops_at_its_face():
    s = _scene([WALL, ((-5.0, 0.0, 0.0), (0.5, 0.5, 0.5), ID)])   # the fast body is body 2
    t, c = _one(s, _entry(2, 0.45), (-5.0, 0.0, 0.0), (10.0, 0.0, 0.0))
    assert c == 0 and abs(t - 0.445) < 1e-6
    tt, col, pos = ccd_ref.step(s, _entry(2, 0.45), [(-5.0, 0.0, 0.0)], [(600.0, 0.0, 0.0)], 1.0 / 60.0, [True])
    assert col[0] == 0 and abs(pos[0, 0] - (-0.55)) < 1e-5 and pos[0, 0] < -0.1   # the centre stays before the near face
    assert pos.dtype == np.float32 and pos[0, 0] == np.float32(-5.0) + (np.float32(600.0) * np.float32(1.0 / 60.0)) * tt[0]


def test_a_wall_turned_about_the_motion_axis_clamps_at_the_same_face():
    q = (float(np.sin(np.pi / 8)), 0.0, 0.0, float(np.cos(np.pi / 8)))   # 45 degrees about x
    s = _scene([((0.0, 0.0, 0.0), (0.1, 2.0, 2.0), q), ((-5.0, 0.0, 0.0), (0.5, 0.5, 0.5), ID)])
    t, c = _one(s, _entry(2, 0.45), (-5.0, 0.0, 0.0), (10.0, 0.0, 0.0))
    assert c == 0 and abs(t - 0.445) < 1e-6


def test_a_sphere_target():
    s = _scene([((-5.0, 0.0, 0.0), (0.5, 0.5, 0.5), ID)], [((0.0, 0.0, 0.0), 1.0)])
    t, c = _one(s, _entry(1, 0.5), (-5.0, 0.0, 0.0), (10.0, 0.0, 0.0))
    assert c == 1 and abs(t - 0.35) < 1e-6


def test_the_closer_of_two_walls_whatever_their_order():
    far, near = ((2.0, 0.0, 0.0), (0.1, 2.0, 2.0), ID), WALL
    for walls, want in (([near, far], 0), ([far, near], 1)):
        s = _scene(walls + [((-5.0, 0.0, 0.0), (0.5, 0.5, 0.5), ID)])
        t, c = _one(s, _entry(3, 0.45), (-5.0, 0.0, 0.0), (10.0, 0.0, 0.0))
        assert c == want and abs(t - 0.445) < 1e-6


def test_ties_go_to_the_smaller_collider_index():
    s = _scene([WALL, WALL, ((-5.0, 0.0, 0.0), (0.5, 0.5, 0.5), ID)])
    assert _one(s, _entry(3, 0.45), (-5.0, 0.0, 0.0), (10.0, 0.0, 0.0))[1] == 0
    s = _scene([((-5.0, 0.0, 0.0), (0.5, 0.5, 0.5), ID)], [((0.0, 0.0, 0.0), 1.0), ((0.0, 0.0, 0.0), 1.0)])
    t, c = _one(s, _entry(1, 0.5), (-5.0, 0.0, 0.0), (10.0, 0.0, 0.0))
    assert c == 1 and abs(t - 0.35) < 1e-6


def test_a_collider_touched_at_the_start_is_skipped_while_a_farther_one_clamps():
    ground = ((0.0, -1.0, 0.0), (20.0, 0.5, 20.0), ID)   # top face at y = -0.5, the sphere rests on it
    s = _scene([ground, ((5.0, 0.0, 0.0), (0.1, 2.0, 2.0), ID), ((0.0, 0.0, 0.0), (0.5, 0.5, 0.5), ID)])
    t, c = _one(s, _entry(3, 0.5), (0.0, 0.0, 0.0), (10.0, 0.0, 0.0))
    assert c == 1 and abs(t - 0.44) < 1e-6
    t, c = _one(s, _entry(3, 0.5), (0.0, 0.0, 0.0), (-10.0, 0.0, 0.0))   # sliding away along the ground: no clamp
    assert (t, c) == (1.0, ccd_ref.NO_HIT)
    t, c = _one(s, _entry(3, 0.5), (0.0, 0.0, 0.0), (10.0, 0.0, 0.0), start_skip=False)   # nb_shapecast's rule: the ground at t = 0
    assert (t, c) == (0.0, 0)


def test_the_threshold_is_strict_and_infinity_never_casts():
    s = _scene([WALL, ((-5.0, 0.0, 0.0), (0.5, 0.5, 0.5), ID)])
    p, v, dt = [(-5.0, 0.0, 0.0)], [(20.0, 0.0, 0.0)], 0.5   # d = (10, 0, 0), |d|^2 = 100 exactly
    for thr, clamped in ((10.0, False), (float(np.nextafter(f(10.0), f(0.0))), True), (0.0, True), (INF, False), (1e30, False)):
        t, c, pos = ccd_ref.step(s, _entry(2, 0.45, thr), p, v, dt, [True])
        assert (c[0] == 0) == clamped, thr
        if not clamped:
            assert t[0] == 1.0 and pos[0, 0] == np.float32(5.0)
    t, c, pos = ccd_ref.step(s, _entry(2, 0.45), p, v, dt, [False])   # a body the step does not advance is never clamped nor moved
    assert c[0] == ccd_ref.NO_HIT and pos[0, 0] == np.float32(-5.0)
    t, c, pos = ccd_ref.step(s, _entry(2, 0.45), p, [(0.0, 0.0, 0.0)], dt, [True])   # no motion: an invalid sweep
    assert c[0] == ccd_ref.NO_HIT and pos[0, 0] == np.float32(-5.0)


def test_filters_apply_both_ways():
    filt = np.zeros(2, scenes.FILTER)
    filt["category"], filt["mask"] = (0x0002, 0x0001), (0xffff, 0xffff)   # the wall is category 2 and collides with everything
    s = _scene([WALL, ((-5.0, 0.0, 0.0), (0.5, 0.5, 0.5), ID)], filters=filt)
    go = lambda e, fl: _one(s, e, (-5.0, 0.0, 0.0), (10.0, 0.0, 0.0), filters=fl)[1]
    assert go(_entry(2, 0.45), filt) == 0
    assert go(_entry(2, 0.45, mask=0x0001), filt) == ccd_ref.NO_HIT          # the entry's mask excludes the wall's category
    filt2 = filt.copy(); filt2["mask"][0] = 0x0004
    assert go(_entry(2, 0.45, category=0x0001), filt2) == ccd_ref.NO_HIT   # the wall's mask excludes the entry's category
    assert go(_entry(2, 0.45, category=0x0004), filt2) == 0
    assert go(_entry(2, 0.45, category=0x0004), None) == 0                 # no table: every collider word is NB_FILTER_ALL


def test_the_connected_skip_sensors_and_the_own_body():
    s = _scene([WALL, ((-5.0, 0.0, 0.0), (0.5, 0.5, 0.5), ID)])
    go = lambda sc, **kw: _one(sc, _entry(2, 0.45), (-5.0, 0.0, 0.0), (10.0, 0.0, 0.0), **kw)[1]
    assert go(s) == 0 and go(s, connected=[(1, 2)]) == ccd_ref.NO_HIT and go(s, connected=[(2, 1)]) == ccd_ref.NO_HIT
    assert go(s, connected=[(1, 3)]) == 0
    sen = _scene([WALL, ((-5.0, 0.0, 0.0), (0.5, 0.5, 0.5), ID)], sensors=np.array([1, 0], np.uint8))
    assert go(sen) == ccd_ref.NO_HIT
    own = _scene([(WALL[0], WALL[1], WALL[2], 2), ((-5.0, 0.0, 0.0), (0.5, 0.5, 0.5), ID)])   # the wall belongs to the fast body
    assert go(own) == ccd_ref.NO_HIT


def _random_scene(rng, nb=60, ns=40):
    boxes = [(tuple(rng.uniform(-8, 8, 3)), tuple(rng.uniform(0.1, 1.5, 3)), tuple(q)) for q in
             (lambda a: a / np.linalg.norm(a, axis=1, keepdims=True))(rng.normal(size=(nb, 4)))]
    spheres = [(tuple(rng.uniform(-8, 8, 3)), float(rng.uniform(0.1, 1.5))) for _ in range(ns)]
    return _scene(boxes, spheres)


def test_without_the_start_skip_the_hits_are_the_shape_casts_and_at_radius_0_the_rays():
    rng = np.random.default_rng(7)
    for _ in range(3):
        s = _random_scene(rng)
        n = 200
        body = rng.integers(1, len(s.body) + 1, n).astype(np.uint32)
        p = rng.uniform(-10, 10, (n, 3)).astype(f)
        d = rng.uniform(-12, 12, (n, 3)).astype(f)
        for radius in (0.0, 0.3, 1.0):
            e = np.zeros(n, abi.CCD_BODY)
            e["body"], e["radius"], e["category"], e["mask"] = body, radius, 0xffff, 0xffff
            t, c = ccd_ref.cast(s, e, p, d, start_skip=False)
            casts = np.zeros(n, abi.SHAPE_CAST)
            q = casts["shape"]
            q["shape"], q["center"], q["radius"], q["mask"], q["ignore_body"] = abi.OVERLAP_SPHERE, p, radius, 0xffffffff, body
            q["rotation"][:, 3] = 1.0
            casts["direction"], casts["max_t"] = d, 1.0
            ref = shapecast_ref.cast(s, casts)
            assert (c == ref["collider"]).all()
            hit = c != ccd_ref.NO_HIT
            assert hit.sum() > 20 and (t[hit].view(np.uint32) == ref["t"][hit].view(np.uint32)).all() and (t[~hit] == 1.0).all()
            if radius == 0.0:
                rays = np.zeros(n, abi.RAY)
                rays["origin"], rays["direction"], rays["max_t"], rays["mask"], rays["ignore_body"] = p, d, 1.0, 0xffffffff, body
                rr = raycast_ref.cast(s, rays)
                assert (c == rr["collider"]).all() and (t[hit].view(np.uint32) == rr["t"][hit].view(np.uint32)).all()


def test_ccd_body_layout_matches_the_header(tmp_path):
    dt, name = abi.CCD_BODY, "nb_ccd_body"
    src = tmp_path / "layout.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "nudge_b200.h"\nint main(void) {\n' +
                   "".join('printf("%%zu\\n", offsetof(%s, %s));\n' % (name, k) for k in dt.names) +
                   'printf("%%zu\\n", sizeof(%s)); return 0; }\n' % name)
    exe = tmp_path / "layout"
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), "-o", str(exe), str(src)])
    out = [int(x) for x in subprocess.check_output([str(exe)]).split()]
    assert out == [dt.fields[k][1] for k in dt.names] + [16]


def test_a_sphere_clamped_onto_a_face_moves_away_and_along_it_next_step():
    """Walls of random, non-round half extents hit by spheres of random radius: the clamp puts the centre on the face slab, where the
    slab may count a start as inside while step 0, rounded the other way, does not.  From the clamped pose the next cast away from the wall
    or along its face must not hit it, and one into it must (at once)."""
    rng = np.random.default_rng(21)
    n = 2000
    stuck_before = 0
    for k in range(n):
        h = (float(rng.uniform(0.05, 0.5)), float(rng.uniform(1.0, 3.0)), float(rng.uniform(1.0, 3.0)))
        q = ID if k % 2 else tuple((lambda a: a / np.linalg.norm(a))(np.array([rng.uniform(-0.5, 0.5), 0.0, 0.0, 1.0])))
        r = float(rng.uniform(0.05, 0.45))
        s = _scene([((0.0, 0.0, 0.0), h, q), ((-5.0, 0.0, 0.0), (0.5, 0.5, 0.5), ID)])
        p0, d0 = np.array([-5.0, rng.uniform(-0.3, 0.3), rng.uniform(-0.3, 0.3)], f), np.array([rng.uniform(8.0, 12.0), 0.0, 0.0], f)
        t, c = _one(s, _entry(2, r), p0, d0)
        assert c == 0, k
        pc = p0 + d0 * f(t)
        for d in ((-3.0, 0.0, 0.0), (0.0, 0.3, 0.0), (0.0, 0.0, -0.3)):   # along the face: staying inside its extent
            assert _one(s, _entry(2, r), pc, d)[1] == ccd_ref.NO_HIT, (k, h, r, d)
        # into the wall: a t = 0 hit, unless step 0 holds (then nb_collide's contact stops the body)
        start = overlap_ref._sphere_box(tuple(f(x) for x in pc), f(r), *(tuple(np.float32([v]) for v in a) for a in
                                        (s.world["position"][0], s.world["rotation"][0], s.half[0])))[0]
        t1, c1 = _one(s, _entry(2, r), pc, (3.0, 0.0, 0.0))
        assert (t1, c1) == (1.0, ccd_ref.NO_HIT) if start else (c1 == 0 and t1 < 1e-5), (k, t1, c1)
        # the touch the face slab finds at t = 0 although step 0 does not hold: a clamp forever without the direction rule
        stuck_before += int(not start and _one(s, _entry(2, r), pc, (-3.0, 0.0, 0.0), start_skip=False) == (0.0, 0))
    assert stuck_before > n // 50, stuck_before
