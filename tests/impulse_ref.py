"""Restatement of body impulses (nb_apply_body_impulses, nb_apply_radial_impulse; DESIGN.md section 8.9): the edit a reference application
makes to its host BodyData between two calls, in numpy float32 with the operation order include/nudge_b200.h specifies (left to right, no
fused multiply-add).  It edits the host arrays of an abi.HostState in place: an OracleSim's BodyData, or a Sim's downloaded rows (then
upload_bodies() sends them back)."""
import numpy as np
from nudge_b200 import scenes

F = np.float32


def world_inverse_inertia(rotation, properties):
    """(n, 6) float32: xx, yy, zz, xy, xz, yz of R diag(inertia_inverse) R^T, in k_inertia's order (nudge.cpp:4182-4199, qmatrix
    nudge.cpp:1142-1163).  rotation (n, 4) x, y, z, w; properties PROPERTIES rows."""
    q = np.asarray(rotation, F).reshape(-1, 4)
    x, y, z, w = q[:, 0], q[:, 1], q[:, 2], q[:, 3]
    kx, ky, kz = x + x, y + y, z + z
    xx, yy, zz = kx * x, ky * y, kz * z
    xy, xz, yz = kx * y, kx * z, ky * z
    sx, sy, sz = kx * w, ky * w, kz * w
    one = F(1.0)
    c0 = (one - yy - zz, xy + sz, xz - sy)
    c1 = (xy - sz, one - xx - zz, yz + sx)
    c2 = (xz + sy, yz - sx, one - xx - yy)
    inv = np.asarray(properties["inertia_inverse"], F).reshape(-1, 3)
    ix, iy, iz = inv[:, 0], inv[:, 1], inv[:, 2]
    e = lambda r, s: ix * c0[r] * c0[s] + iy * c1[r] * c1[s] + iz * c2[r] * c2[s]
    return np.stack([e(0, 0), e(1, 1), e(2, 2), e(0, 1), e(0, 2), e(1, 2)], 1).astype(F)


def apply_body_impulses(state, rows):
    """nb_apply_body_impulses on the host arrays of `state`: every entry in list order."""
    rows = np.asarray(rows, scenes.BODY_IMPULSE).reshape(-1)
    for r in rows:
        b = int(r["body"])
        W = world_inverse_inertia(state.transforms["rotation"][b:b + 1], state.properties[b:b + 1])[0]
        xx, yy, zz, xy, xz, yz = (F(c) for c in W)
        m = F(state.properties["mass_inverse"][b])
        o, J, L = (np.asarray(r[f], F) for f in ("offset", "impulse", "angular_impulse"))
        v = state.momentum["velocity"][b]
        for k in range(3):
            v[k] = v[k] + m * J[k]
        t = (o[1] * J[2] - o[2] * J[1] + L[0], o[2] * J[0] - o[0] * J[2] + L[1], o[0] * J[1] - o[1] * J[0] + L[2])
        w = state.momentum["angular_velocity"][b]
        w[0] = w[0] + ((xx * t[0] + xy * t[1]) + xz * t[2])
        w[1] = w[1] + ((xy * t[0] + yy * t[1]) + yz * t[2])
        w[2] = w[2] + ((xz * t[0] + yz * t[1]) + zz * t[2])
        state.momentum["velocity"][b] = v; state.momentum["angular_velocity"][b] = w
        state.idle[b] = 0


def radial_hits(state, center, radius, kinematic=()):
    """(hit mask over the bodies, d, dist): every body 1..B-1 that is not kinematic and whose position is closer than `radius`."""
    p = np.asarray(state.transforms["position"], F)
    d = p - np.asarray(center, F)
    dist = np.sqrt((d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2])
    hit = dist < F(radius)
    hit[0] = False
    hit[np.asarray(kinematic, np.int64)] = False
    return hit, d, dist


def apply_radial_impulse(state, center, radius, impulse, kinematic=()):
    """nb_apply_radial_impulse on the host arrays of `state`; `kinematic` lists the context's kinematic bodies."""
    hit, d, dist = radial_hits(state, center, radius, kinematic)
    state.idle[hit] = 0
    push = hit & (dist > F(0.0))
    with np.errstate(divide="ignore", invalid="ignore"):
        k = (F(impulse) * (F(1.0) - dist / F(radius))) / dist
    m = state.properties["mass_inverse"].astype(F)
    v = state.momentum["velocity"]
    for c in range(3):
        v[push, c] = v[push, c] + m[push] * (d[push, c] * k[push])
    return hit


def random_impulses(rng, bodies, n, scale=2.0, duplicates=True, zeros=0.2):
    """n BODY_IMPULSE rows on `bodies` (drawn with repetition when `duplicates`), some with zero impulses, off-centre offsets."""
    bodies = np.asarray(bodies)
    r = np.zeros(n, scenes.BODY_IMPULSE)
    r["body"] = rng.choice(bodies, n, replace=duplicates or n > len(bodies))
    r["offset"] = rng.uniform(-0.6, 0.6, (n, 3)) * (rng.random((n, 1)) < 0.7)
    r["impulse"] = rng.normal(0.0, scale, (n, 3))
    r["angular_impulse"] = rng.normal(0.0, 0.5 * scale, (n, 3)) * (rng.random((n, 1)) < 0.5)
    z = rng.random(n) < zeros
    r["impulse"][z] = 0; r["angular_impulse"][z] = 0
    return r
