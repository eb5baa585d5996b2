"""The broadphase edge-case scenes shared by tests/test_broadphase_ref.py (CPU: oracle against brute force and the reference) and
tests/test_gpu_broadphase_edges.py (GPU against the oracle): scenes where the grid's cell-fit rule (DESIGN.md section 2.3) is tight.

Every family is seeded and deterministic.  Each builder returns an EdgeScene: the Scene plus what the test asserts about its grid
(tests/grid_ref.py) before it trusts a comparison.  Builders that have to search (the tight pair, the level boundary, the wrapped corners)
take `rcp`, the rcpps model: Sim.device_rcp on a GPU, grid_ref.host_rcp() on a CPU; both give the same scene on one machine."""
import numpy as np
from nudge_b200 import scenes
from tests import grid_ref as G

f = np.float32


class EdgeScene:
    def __init__(self, name, scene, kind="plain", **premise):
        self.name, self.scene, self.kind, self.premise = name, scene, kind, premise


def pile(n, seed, offset=(0.0, 0.0, 0.0), ground=True, half=10.0, sizes=(0.3, 0.9), rotate=True):
    """n boxes on a jittered lattice in a 10 m square over a ground of half extent `half` (its min corner is the frame's), all moved by
    `offset`.  Body 0 carries the ground (collider 0)."""
    rng = np.random.default_rng(seed)
    side = max(1, int(np.ceil(np.sqrt(n / 3.0))))
    k = np.arange(n)
    pos = np.stack([(k % side) * 2.0 - side + 1.0, (k // (side * side)) * 2.0 + 1.2, ((k // side) % side) * 2.0 - side + 1.0], 1)
    pos = pos + rng.uniform(-0.3, 0.3, pos.shape)
    size = rng.uniform(sizes[0], sizes[1], (n, 3))
    rot = scenes._random_unit_quaternions(rng, n) if rotate else None
    s = scenes._assemble("pile", size.astype(np.float32), pos.astype(np.float32), rot, np.zeros(0, np.float32), np.zeros((0, 3), np.float32),
                         ground=ground, ground_half=(half, 1.0, half), ground_y=-1.0)
    return moved(s, offset)


def moved(s, offset):
    off = np.asarray(offset, np.float64)
    s.transforms["position"][1:] = (s.transforms["position"][1:] + off).astype(np.float32)
    for t in (s.box_transforms, s.sphere_transforms):
        w = t["body"] == 0
        t["position"][w] = (t["position"][w] + off).astype(np.float32)
    return s


def with_spheres(s, centres, radii):
    """Scene s plus one dynamic sphere body per centre; tags stay distinct (boxes first, then spheres)."""
    c = np.asarray(centres, np.float32).reshape(-1, 3); r = np.asarray(radii, np.float32).reshape(-1)
    n0, m = s.n_bodies, len(c)
    t = scenes.Scene(n0 + m, s.n_boxes, s.n_spheres + m)
    for k in ("box_data", "box_transforms", "time_step", "iterations", "gravity", "damping"):
        setattr(t, k, getattr(s, k))
    t.transforms[:n0] = s.transforms; t.properties[:n0] = s.properties; t.momentum[:n0] = s.momentum; t.idle[:n0] = s.idle
    t.transforms["position"][n0:] = c
    t.properties[n0:] = scenes._sphere_props(r)
    t.sphere_data[:s.n_spheres] = s.sphere_data; t.sphere_transforms[:s.n_spheres] = s.sphere_transforms
    t.sphere_data["radius"][s.n_spheres:] = r
    t.sphere_transforms["body"][s.n_spheres:] = n0 + np.arange(m, dtype=np.uint32)
    t.box_tags[:] = np.arange(t.n_boxes, dtype=np.uint32)
    t.sphere_tags[:] = t.n_boxes + np.arange(t.n_spheres, dtype=np.uint32)
    t.connections = s.connections
    t.name = s.name
    return t


def with_boxes(s, centres, halves):
    """Scene s plus boxes at `centres` with half extents `halves`, each on a new dynamic body."""
    c = np.asarray(centres, np.float32).reshape(-1, 3); h = np.asarray(halves, np.float32).reshape(-1, 3)
    m = len(c)
    nb0, n0 = s.n_boxes, s.n_bodies
    t = scenes.Scene(n0 + m, nb0 + m, s.n_spheres)
    for k in ("sphere_data", "sphere_transforms", "time_step", "iterations", "gravity", "damping"):
        setattr(t, k, getattr(s, k))
    t.transforms[:n0] = s.transforms; t.properties[:n0] = s.properties; t.momentum[:n0] = s.momentum; t.idle[:n0] = s.idle
    t.box_data[:nb0] = s.box_data; t.box_transforms[:nb0] = s.box_transforms
    t.box_data["size"][nb0:] = h
    t.transforms["position"][n0:] = c
    t.properties[n0:] = scenes._box_props(h)
    t.box_transforms["body"][nb0:] = n0 + np.arange(m, dtype=np.uint32)
    t.box_tags[:] = np.arange(t.n_boxes, dtype=np.uint32)
    t.sphere_tags[:] = t.n_boxes + np.arange(t.n_spheres, dtype=np.uint32)
    t.connections = s.connections
    t.name = s.name
    return t


def _ulps(x, k):
    """x moved by k float32 ulps (k may be negative)."""
    x = f(x)
    for _ in range(abs(k)):
        x = np.nextafter(x, f(np.inf) if k > 0 else f(-np.inf))
    return x


# ---------------- far from the origin ----------------
FAR_EXPONENTS = (16, 20, 24, 26, 28)


def far(e, rcp):
    """A pile with its own ground, moved so that |smin * L| is about 2^e, plus the tightest pair the cell-fit rule allows: sphere a passes
    the small test at the grid level with the largest radius it can, its min corner sits in the last quantised unit of a cell (searched ulp
    by ulp) so that its far face lies in the next cell, and sphere b's min corner sits one float below a's max corner."""
    base = pile(150, seed=e)
    g0 = G.Grid.of_scene(base, rcp)
    d = 2.0 ** e / float(g0.frame.L[0])
    s = pile(150, seed=e, offset=(d, d, d))
    g = G.Grid.of_scene(s, rcp)
    L, j = float(g.frame.L[0]), g.j
    W = 1 << j
    # the spheres sit beside the pile, inside the frame of min corners, so L and j stay as they are
    y, z = f(d + 4.0), f(d - 6.0)
    r0 = f((W - 2) / L / 2.0 * (1 + 1e-5))
    box = lambda p, r: (np.array([[p - r, y - r, z - r]], np.float32), np.array([[p + r, y + r, z + r]], np.float32))
    best = None
    for cell_x in range(2, 5):
        x_lo = (cell_x * W + W - 0.5 + float(g.frame.ms[0])) / L   # the last unit of cell cell_x
        pa0 = f(x_lo + float(r0))
        for k in range(-48, 49):
            pa = _ulps(pa0, k)
            r = r0
            while G.level_needed(*box(pa, r), L)[0] > j:   # the largest radius that still passes at this position
                r = np.nextafter(r, f(0))
            lo, hi = box(pa, r)
            q0, q1 = g.frame.quantise(lo)[0, 0], g.frame.quantise(hi)[0, 0]
            if q0 >> j != cell_x or q1 >> j != cell_x + 1:
                continue
            key = (int(q1) - int(q0), float(hi[0, 0] - lo[0, 0]))
            if best is None or key > best[0]:
                best = (key, pa, r, hi[0, 0])
    (span, _), pa, ra, ahi = best
    rb = f(0.25)
    pb = f(ahi + rb)
    while not f(pb - rb) < ahi:
        pb = np.nextafter(pb, f(-np.inf))
    while f(np.nextafter(pb, f(np.inf)) - rb) < ahi:
        pb = np.nextafter(pb, f(np.inf))
    t = with_spheres(s, [(pa, y, z), (pb, y, z)], [ra, rb])
    t.name = "far_2^%d" % e
    a = t.n_colliders - 2
    return EdgeScene(t.name, t, scaled_min=(2.0 ** (e - 1), 2.0 ** (e + 1)), tight_pair=(a, a + 1), level=j)


# ---------------- level boundary ----------------
def boundary(side, n_b, rcp):
    """A pile plus an 8 x 8 layer of n_b spheres (neighbours overlap by a little, inside the frame the ground's min corner spans, so L stays
    as it is) whose quantised extent sits at the boundary of level l, one above the pile's: side "at" = the largest radius with
    extent * L + 2 <= 2^l, "below" / "above" = one ulp smaller / larger.  The pile has more than 64 colliders of its own that need level l, so
    "at" and "below" spheres are small at j = l with their span at the cell-fit bound.  "above" spheres need l + 1: 63 of them and the ground
    are exactly 64 colliders too large for level l, so the grid stays at l and they go through k_large_pairs; with 64 of them the grid moves
    up to l + 1 and they are small there."""
    assert n_b <= 64
    s = pile(300, seed=31, half=30.0)
    g = G.Grid.of_scene(s, rcp)
    L, l = float(g.frame.L[0]), g.j + 1
    cx, cy, cz = [], [], []
    r0 = f((2 ** l - 2) / L / 2.0)
    radii = []
    for i in range(n_b):
        x, y, z = f(-25.0 + (i % 8) * 2.0 * float(r0) * 0.999), f(14.0), f(-25.0 + (i // 8) * 2.0 * float(r0) * 0.999)
        r = r0
        ok = lambda r: G.level_needed(np.array([[x - r, y - r, z - r]], np.float32), np.array([[x + r, y + r, z + r]], np.float32), L)[0] <= l
        while not ok(r):
            r = np.nextafter(r, f(0))
        while ok(np.nextafter(r, f(np.inf))):
            r = np.nextafter(r, f(np.inf))
        r = {"at": r, "below": np.nextafter(r, f(0)), "above": np.nextafter(r, f(np.inf))}[side]
        cx.append(x); cy.append(y); cz.append(z); radii.append(r)
    t = with_spheres(s, np.stack([cx, cy, cz], 1), radii)
    t.name = "boundary_%s_%d" % (side, n_b)
    first = t.n_colliders - n_b
    above = side == "above"
    # (first sphere, the level the spheres need, the grid level, whether the spheres are small)
    return EdgeScene(t.name, t, boundary=(first, l + above, l + (above and n_b == 64), not above or n_b == 64))


# ---------------- large colliders ----------------
LARGE_COUNTS = (63, 64, 65, 200)


def large(n, variant="dynamic"):
    """A field of small boxes under n - 1 large slabs (half extents 3 x 0.2 x 3, level above the boxes'), so that with the ground n
    colliders need the coarser level: at n <= 64 they go through k_large_pairs, above that the grid moves up.  Slabs overlap each other
    (large against large) and the boxes.  variant "features": some slabs filtered by category, two of them sensor zones, and, with the
    connected opt-out, a slab's body connected to the body of a box it overlaps and two overlapping slabs' bodies connected (premise
    "connected": each connection removes at least one pair that nothing else would); "kinematic": every fourth slab on a kinematic body, two
    of them moving."""
    rng = np.random.default_rng(100 + n)
    s = pile(400, seed=n, half=30.0)
    m = n - 1
    c = np.stack([rng.uniform(-7, 7, m), 1.5 + (np.arange(m) % 12) * 0.35 + rng.uniform(0, 0.1, m), rng.uniform(-7, 7, m)], 1)
    t = with_boxes(s, c, np.tile([[3.0, 0.2, 3.0]], (m, 1)))
    t.name = "large_%d_%s" % (n, variant)
    slabs = np.arange(t.n_boxes - m, t.n_boxes)
    bodies = t.box_transforms["body"][slabs].astype(np.int64)
    es = EdgeScene(t.name, t, kind=variant, large_count=n, slabs=slabs)
    if variant == "features":
        k = t.n_colliders
        filt = np.zeros(k, scenes.FILTER); filt["category"] = 1; filt["mask"] = 0xffff
        filt["category"][slabs[::3]] = 2; filt["mask"][slabs[::3]] = 0xfffe            # no slab of these touches a box or the ground
        filt["category"][slabs[1::5]] = 4; filt["mask"][slabs[1::5]] = 0x4 | 0x1      # these skip other categories' slabs
        t.collision_filters = filt
        t.filter_flags = scenes.FILTER_SKIP_CONNECTED
        sens = np.zeros(k, np.uint8); sens[slabs[2]] = 1; sens[slabs[7]] = 1
        t.sensors = sens
        # connect overlapping pairs that pass the category filter and hold no sensor: a slab and a box, and two slabs
        plain = (filt["category"] == 1) & (sens == 0)
        body = t.box_transforms["body"].astype(np.int64)
        lo, hi = G.scene_aabbs(t)
        cand = sorted((a, b) for a, b in G.brute_pairs(lo, hi) if plain[a] and plain[b] and body[a] != body[b] and a > 0)
        slab = set(slabs.tolist())
        box_slab = next((a, b) for a, b in cand if (a in slab) != (b in slab))
        slab_slab = next((a, b) for a, b in cand if a in slab and b in slab)
        t.connections = np.array([(body[a], body[b]) for a, b in (box_slab, slab_slab)], scenes.PAIR32)
        es.premise["connected"] = (box_slab, slab_slab)
    elif variant == "kinematic":
        kin = bodies[::4]
        rows = np.zeros(len(kin), scenes.KINEMATIC); rows["body"] = kin
        rows["velocity"][0] = (0.5, 0.0, 0.0); rows["velocity"][1] = (0.0, 0.3, 0.0); rows["angular_velocity"][1] = (0.0, 0.2, 0.0)
        t.kinematic = rows
    return es


# ---------------- one cell ----------------
def one_cell(over):
    """A pile under 70 thin boards that each span the whole frame of min corners: their extent needs level 16 (over = False) or more
    than any level (over = True), so more than 64 colliders need level 16 and the grid is a single cell."""
    s = pile(300, seed=41 + over)
    lo = G.scene_aabbs(s)[0]
    span = float(lo[:, 0].max() - lo[:, 0].min())
    hx = span * (0.85 if over else 0.3)
    rng = np.random.default_rng(7)
    c = np.stack([rng.uniform(-2, 2, 70), 12.0 + np.arange(70) * 0.09, rng.uniform(-6, 6, 70)], 1)
    t = with_boxes(s, c, np.tile([[hx, 0.05, 0.6]], (70, 1)))
    t.name = "one_cell_%s" % ("beyond" if over else "level16")
    return EdgeScene(t.name, t, level=16)


# ---------------- degenerate frames ----------------
def flat_layer():
    """Spheres of one radius resting at one height, no ground: the y range of the min corners is 0."""
    rng = np.random.default_rng(51)
    n = 200
    p = np.stack([rng.uniform(-6, 6, n), np.full(n, 3.0), rng.uniform(-6, 6, n)], 1)
    s = scenes._assemble("flat_layer", np.zeros((0, 3), np.float32), np.zeros((0, 3), np.float32), None, np.full(n, 0.5, np.float32),
                         p.astype(np.float32), ground=False)
    return EdgeScene(s.name, s, flat_axis=1)


def same_corner(n):
    """n boxes of one size at one position: every min corner equal, so L is infinite and every collider is large."""
    s = scenes._assemble("same_corner_%d" % n, np.full((n, 3), 0.5, np.float32), np.tile([[1.0, 2.0, 3.0]], (n, 1)).astype(np.float32), None,
                         np.zeros(0, np.float32), np.zeros((0, 3), np.float32), ground=False)
    return EdgeScene(s.name, s, all_large=True)


def few(n):
    """One box, or two overlapping boxes, alone."""
    pos = np.array([[0.0, 1.0, 0.0], [0.6, 1.5, 0.3]], np.float32)[:n]
    s = scenes._assemble("alone_%d" % n, np.full((n, 3), 0.5, np.float32), pos, None, np.zeros(0, np.float32), np.zeros((0, 3), np.float32),
                         ground=False)
    return EdgeScene(s.name, s)


# ---------------- wrapped corners ----------------
def wrapped(rcp):
    """A pile whose x range of min corners R is a float where rcpps overestimates 1 / R, so that 65535 * rcp(R) * R > 65536: the colliders
    whose min corner is the scene's largest x quantise past 65535 and are large.  Five spheres sit there, overlapping each other and a box."""
    s = pile(200, seed=61, half=6.0)
    g = G.Grid.of_scene(s, rcp)
    lo_x = float(g.frame.smin[0])
    base = f(g.frame.smax[0] - g.frame.smin[0] + 2.0)
    cand = np.array([_ulps(base, 4096 * k) for k in range(64)], np.float32)
    over = (f(65535.0) * rcp(cand)).astype(np.float64) * cand.astype(np.float64)
    R = cand[int(np.argmax(over))]
    r = f(0.4)
    xs = f(f(lo_x) + R)
    centres = [(xs + r, 2.0 + 0.7 * i, 0.5 * i) for i in range(5)]
    t = with_spheres(s, np.array(centres, np.float32), np.full(5, r, np.float32))
    # the sphere centres are rounded: put each min corner exactly on lo_x + R
    for i in range(5):
        p = t.transforms["position"][t.n_bodies - 5 + i]
        while f(p[0] - r) > xs:
            p[0] = np.nextafter(p[0], f(-np.inf))
        while f(p[0] - r) < xs:
            p[0] = np.nextafter(p[0], f(np.inf))
    t.name = "wrapped"
    return EdgeScene(t.name, t, wrapped=np.arange(t.n_colliders - 5, t.n_colliders))


# ---------------- multi-scale ----------------
def multi_scale(seed=71):
    """Rotated boxes and spheres with log-uniform half extents from 2^-6 to 2^5 over a ground."""
    rng = np.random.default_rng(seed)
    nb, ns = 400, 400
    size = np.exp2(rng.uniform(-6, 5, (nb, 1)) + rng.uniform(-0.5, 0.5, (nb, 3))).clip(2.0 ** -6, 32.0)
    rad = np.exp2(rng.uniform(-6, 5, ns))
    pos = lambda k: np.stack([rng.uniform(-60, 60, k), rng.uniform(0, 60, k), rng.uniform(-60, 60, k)], 1).astype(np.float32)
    s = scenes._assemble("multi_scale", size.astype(np.float32), pos(nb), scenes._random_unit_quaternions(rng, nb), rad.astype(np.float32), pos(ns),
                         ground_half=(120.0, 1.0, 120.0), ground_y=-1.0)
    return EdgeScene(s.name, s)


CAPACITY = 1 << 17   # contacts: the multi-scale scene's largest boxes touch many others


def input_digest(s):
    """Digest of everything a step of the reference reads from scene s."""
    from tests.parity_util import digest
    parts = [s.transforms, s.properties, s.momentum, s.idle, s.box_tags, s.box_data, s.box_transforms, s.sphere_tags, s.sphere_data,
             s.sphere_transforms, s.connections]
    return digest(np.frombuffer(b"".join(np.ascontiguousarray(p).tobytes() for p in parts), np.uint8))


def all_scenes(rcp):
    """Every family, in a fixed order."""
    out = [far(e, rcp) for e in FAR_EXPONENTS]
    out += [boundary(side, n, rcp) for side in ("at", "below", "above") for n in (63, 64)]
    out += [large(n) for n in LARGE_COUNTS]
    out += [large(n, v) for n in (64, 200) for v in ("features", "kinematic")]
    out += [one_cell(False), one_cell(True), flat_layer(), same_corner(12), few(1), few(2), wrapped(rcp), multi_scale()]
    return out
