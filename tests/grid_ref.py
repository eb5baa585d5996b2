"""numpy restatement of what the grid broadphase decides before it looks for pairs (nudge_b200/csrc/nb_collide.cuh K1-K4) — TEST
INFRASTRUCTURE ONLY.

It restates, operation by operation in float32: the collider AABBs of k_collider_world, the Morton frame (morton_frame: scene bounds over
the AABB min corners, scale L = 65535 * rcp(range), the scaled min corner), the quantisation of a corner (morton_quantise: one fused
multiply-subtract, then truncation), the level a collider needs (grid_level_needed), the level the step picks (grid_setup) and the small
flag of k_grid_build.  rcp is the rcpps model the device and the oracle share: pass Sim.device_rcp on a GPU, or host_rcp() (the oracle's
own rcpps) on a CPU.  brute_pairs is the pair set every broadphase must produce: every strictly overlapping AABB pair.

The grid's one geometric claim (DESIGN.md section 2.3): a small collider's quantised span q(hi) - q(lo) is at most 2^j - 1, so two
overlapping small colliders have min-corner cells at most one apart per axis.  The quantisation rounds once (x * L - ms is fused), so its
error is half an ulp of a value below 65536 whatever the distance from the origin; quantised_span lets a test check the claim directly."""
import numpy as np
from oracle.raycast_ref import world_transforms

f = np.float32
NB_GRID_MAX_LARGE = 64


def host_rcp():
    """The oracle's rcpps (the host CPU's, which the device's table is sampled from)."""
    from oracle import pyoracle
    lib = pyoracle.load()

    def rcp(x):
        x = np.ascontiguousarray(x, np.float32).reshape(-1); y = np.empty_like(x)
        lib.nbo_rcp(x.ctypes.data, y.ctypes.data, len(x))
        return y
    return rcp


def fma32(a, b, c):
    """fmaf(a, b, c) on float32 arrays: a * b + c rounded once.  The product is exact in float64; the sum is made exact with TwoSum and
    rounded to odd in float64, which then rounds to float32 correctly (53 >= 24 + 2 bits)."""
    a, b, c = (np.asarray(x, np.float32).astype(np.float64) for x in (a, b, c))
    with np.errstate(all="ignore"):
        p = a * b
        s = p + c
        bb = s - p
        e = (p - (s - bb)) + (c - bb)
        u = np.array(s, np.float64).view(np.uint64).copy()
        inexact = np.isfinite(e) & (e != 0)
        u[inexact & ((e < 0) != (s < 0))] -= np.uint64(1)   # the exact value lies below |s|: truncate toward zero
        u[inexact] |= np.uint64(1)
        return u.view(np.float64).astype(np.float32)


def toint(x):
    """cvttps2dq then (u32): truncation; out of range or NaN -> 0x80000000."""
    x = np.asarray(x, np.float32)
    with np.errstate(invalid="ignore"):
        ok = (x > f(-2147483904.0)) & (x < f(2147483648.0))
    r = np.full(x.shape, -2 ** 31, np.int64)
    r[ok] = np.trunc(x[ok]).astype(np.int64)
    return (r & 0xffffffff).astype(np.uint32)


def nb_min(x, y):
    return np.where(y < x, y, x)


def aabbs(body_xf, box_xf, box_data, sphere_xf, sphere_data):
    """(lo, hi): the float32 (K, 3) corners k_collider_world writes, boxes then spheres."""
    w = world_transforms(body_xf, box_xf, sphere_xf)
    nb = len(box_xf)
    p = w["position"].astype(np.float32)
    q = w["rotation"][:nb].astype(np.float32)
    x, y, z, s = q[:, 0], q[:, 1], q[:, 2], q[:, 3]
    kx, ky, kz = x + x, y + y, z + z
    xx, yy, zz = kx * x, ky * y, kz * z
    xy, xz, yz = kx * y, kx * z, ky * z
    sx, sy, sz = kx * s, ky * s, kz * s
    one = f(1.0)
    c0 = ((one - yy) - zz, xy + sz, xz - sy)
    c1 = (xy - sz, (one - xx) - zz, yz + sx)
    c2 = (xz + sy, yz - sx, (one - xx) - yy)
    h = box_data["size"].astype(np.float32)
    ext = np.zeros((len(p), 3), np.float32)
    for k in range(3):
        ext[:nb, k] = (np.abs(c0[k] * h[:, 0]) + np.abs(c1[k] * h[:, 1])) + np.abs(c2[k] * h[:, 2])
    ext[nb:] = sphere_data["radius"].astype(np.float32)[:, None]
    return p - ext, p + ext


def scene_aabbs(scene):
    return aabbs(scene.transforms, scene.box_transforms, scene.box_data, scene.sphere_transforms, scene.sphere_data)


class Frame:
    """The Morton frame of a set of min corners (morton_frame): L[4] (lane i & 3 scales collider i), ms[3] = smin * L."""

    def __init__(self, lo, rcp):
        lo = np.asarray(lo, np.float32)
        smin = np.zeros(4, np.float32); smax = np.zeros(4, np.float32)
        smin[:3] = lo.min(axis=0); smax[:3] = lo.max(axis=0)
        with np.errstate(all="ignore"):
            sc = f(65535.0) * np.asarray(rcp(smax - smin), np.float32)
        A = [nb_min(sc[0], sc[2]), nb_min(sc[1], sc[2]), nb_min(sc[2], sc[0]), nb_min(sc[2], sc[1])]
        self.L = np.array([nb_min(A[0], A[1]), nb_min(A[1], A[0]), nb_min(A[2], A[3]), nb_min(A[3], A[2])], np.float32)
        with np.errstate(all="ignore"):
            self.ms = smin[:3] * self.L[:3]
        self.smin, self.smax = smin[:3], smax[:3]

    def quantise(self, corner, index=None):
        """morton_quantise of (K, 3) corners of the colliders with the given original indices (default 0..K-1): uint32 (K, 3)."""
        c = np.asarray(corner, np.float32).reshape(-1, 3)
        idx = np.arange(len(c)) if index is None else np.asarray(index)
        s = self.L[idx & 3]
        return np.stack([toint(fma32(c[:, k], s, -self.ms[k])) for k in range(3)], axis=1)


def level_needed(lo, hi, scale):
    """grid_level_needed: the smallest l in 1..16 with max extent * scale + 2 <= 2^l, 17 if none (also for NaN)."""
    lo = np.asarray(lo, np.float32).reshape(-1, 3); hi = np.asarray(hi, np.float32).reshape(-1, 3)
    d = hi - lo
    with np.errstate(all="ignore"):
        ext = np.fmax(d[:, 0], np.fmax(d[:, 1], d[:, 2])) * f(scale) + f(2.0)
    out = np.full(len(lo), 17, np.int64)
    for l in range(16, 0, -1):
        with np.errstate(invalid="ignore"):
            out[ext <= f(1 << l)] = l
    return out


def grid_setup(levels):
    """The grid level j: the finest level that leaves at most NB_GRID_MAX_LARGE colliders needing a coarser one (16 if none does)."""
    hist = np.bincount(np.asarray(levels, np.int64), minlength=18)
    j, above = 16, int(hist[17])
    for l in range(16, 0, -1):
        if above <= NB_GRID_MAX_LARGE:
            j = l
        above += int(hist[l])
    return j


class Grid:
    """Everything the grid decides for AABBs (lo, hi): frame, quantised corners q_lo / q_hi, levels, j, the small flags, the large count."""

    def __init__(self, lo, hi, rcp):
        self.lo, self.hi = np.asarray(lo, np.float32), np.asarray(hi, np.float32)
        self.frame = Frame(self.lo, rcp)
        self.q_lo = self.frame.quantise(self.lo)
        self.q_hi = self.frame.quantise(self.hi)
        self.levels = level_needed(self.lo, self.hi, self.frame.L[0])
        self.j = grid_setup(self.levels)
        self.small = (self.levels <= self.j) & (self.q_lo < 65536).all(axis=1)
        self.n_large = int((~self.small).sum())

    @classmethod
    def of_scene(cls, scene, rcp):
        return cls(*scene_aabbs(scene), rcp)

    def span(self):
        """q(hi) - q(lo) per collider and axis, as int64 (the quantity the claim bounds by 2^j - 1 for small colliders)."""
        return self.q_hi.astype(np.int64) - self.q_lo.astype(np.int64)

    def cell(self):
        return (self.q_lo >> np.uint32(self.j)).astype(np.int64)

    def max_scaled_min(self):
        """max |smin * L| over the axes: how far the frame's origin lies from the world's, in quantised units."""
        return float(np.abs(self.frame.ms.astype(np.float64)).max())


def brute_pairs(lo, hi):
    """Every strictly overlapping float32 AABB pair, as a set of (i, j) with i < j."""
    lo = np.asarray(lo, np.float32); hi = np.asarray(hi, np.float32)
    K = len(lo)
    out = set()
    for a in range(0, K, 256):
        b = min(K, a + 256)
        hit = np.ones((b - a, K), bool)
        for k in range(3):
            hit &= (hi[None, :, k] > lo[a:b, None, k]) & (hi[a:b, None, k] > lo[None, :, k])
        i, j = np.nonzero(hit)
        i = i + a
        keep = i < j
        out.update(zip(i[keep].tolist(), j[keep].tolist()))
    return out


def pair_set(lo_idx, hi_idx):
    """A pair list (collider indices, either orientation) as a set of (min, max)."""
    a, b = np.asarray(lo_idx, np.int64), np.asarray(hi_idx, np.int64)
    return set(zip(np.minimum(a, b).tolist(), np.maximum(a, b).tolist()))
