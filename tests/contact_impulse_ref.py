"""A numpy restatement of the contact impulse reports (nb_get_body_contact_impulses, nb_get_contact_pair_impulses; include/nudge_b200.h,
DESIGN.md section 8.22), float32 operation by operation in the header's order.

Inputs: the contact set (scenes.CONTACT data, scenes.PAIR32 bodies, uint64 tags) in nb_download_contacts' order, the per-contact world
impulses J_c (n x 3 float32, or nb_debug_read("impulses") rows whose first three words are J_c), the (tag, feature) order
(nb_debug_read("sorted")), and the bodies' positions at the step's start (n_bodies x 3 float32)."""
import numpy as np
from nudge_b200 import abi

f32 = np.float32
REMOVED = 0xffffffff


def _j(impulses):
    a = np.asarray(impulses)
    if a.dtype.names:
        a = a["impulse"]
    return np.ascontiguousarray(np.asarray(a, f32)[:, :3])


def cross(r, j):
    """The header's cross(u, v) per row, float32."""
    return np.stack([r[:, 1] * j[:, 2] - r[:, 2] * j[:, 1], r[:, 2] * j[:, 0] - r[:, 0] * j[:, 2], r[:, 0] * j[:, 1] - r[:, 1] * j[:, 0]], axis=1)


def dot(u, v):
    """The header's dot(u, v) = (u.x*v.x + u.y*v.y) + u.z*v.z per row, float32."""
    return (u[:, 0] * v[:, 0] + u[:, 1] * v[:, 1]) + u[:, 2] * v[:, 2]


def body_report(data, bodies, impulses, positions, n_bodies, idx=None, device=False):
    """nb_get_body_contact_impulses' rows for the indices idx (None: 0 .. n_bodies - 1).  device: an index at or beyond n_bodies gives a
    NB_REMOVED_BODY row of zeros (the host mode refuses such an index instead)."""
    J = _j(impulses)
    n = len(J)
    pos = np.asarray(positions, f32).reshape(-1, 3)
    P = np.asarray(data["position"], f32).reshape(-1, 3)
    # the sides in the order they are summed: contact 0 side a, contact 0 side b, contact 1 side a, ...
    side_body = np.stack([bodies["a"], bodies["b"]], axis=1).reshape(-1).astype(np.int64)
    side_c = np.repeat(np.arange(n), 2)
    valid = side_body < n_bodies
    r = P[side_c] - pos[np.minimum(side_body, max(n_bodies - 1, 0))]
    Js = J[side_c]
    cr = cross(r, Js)
    sign_b = np.tile([False, True], n)
    lin = np.where(sign_b[:, None], Js, -Js)   # acc - J equals acc + (-J) in float32, bit for bit
    ang = np.where(sign_b[:, None], cr, -cr)
    acc = np.zeros((n_bodies + 1, 3), f32); tq = np.zeros((n_bodies + 1, 3), f32)
    k = np.zeros(n_bodies + 1, np.uint32)
    tgt = np.where(valid, side_body, n_bodies)
    np.add.at(acc, tgt, lin)   # unbuffered, in index order: the sequential sum
    np.add.at(tq, tgt, ang)
    np.add.at(k, tgt, 1)
    idx = np.arange(n_bodies, dtype=np.uint32) if idx is None else np.asarray(idx, np.uint32)
    out = np.zeros(len(idx), abi.BODY_CONTACT_IMPULSE)
    ok = idx < n_bodies
    if not device and not ok.all():
        raise ValueError("an index at or beyond the body count")
    b = idx[ok].astype(np.int64)
    out["impulse"][ok] = acc[b]; out["angular_impulse"][ok] = tq[b]; out["contacts"][ok] = k[b]; out["body"][ok] = idx[ok]
    out["body"][~ok] = REMOVED
    return out


def body_report_loop(data, bodies, impulses, positions, b):
    """The same row for one body b, written as the header's loop (the check of body_report's vectorised sums)."""
    J = _j(impulses)
    acc = np.zeros(3, f32); tq = np.zeros(3, f32); k = 0
    p = np.asarray(positions, f32).reshape(-1, 3)[b]
    for c in range(len(J)):
        for side, body in ((0, bodies["a"][c]), (1, bodies["b"][c])):
            if body != b:
                continue
            r = np.asarray(data["position"][c], f32) - p
            cr = cross(r[None], J[c][None])[0]
            if side == 0:
                acc = acc - J[c]; tq = tq - cr
            else:
                acc = acc + J[c]; tq = tq + cr
            k += 1
    return acc, tq, k


def pair_rows(data, bodies, tags, impulses, sorted_idx):
    """Every pair's row, in ascending tags order (before the threshold)."""
    J = _j(impulses)
    srt = np.asarray(sorted_idx, np.int64)
    n = len(srt)
    if n == 0:
        return np.zeros(0, abi.CONTACT_PAIR_IMPULSE)
    t = np.asarray(tags, np.uint64)[srt]
    head = np.ones(n, bool); head[1:] = t[1:] != t[:-1]
    run = np.cumsum(head) - 1
    R = int(run[-1]) + 1
    Js = J[srt]
    nrm = np.asarray(data["normal"], f32)[srt]
    imp = np.zeros((R, 3), f32); nsum = np.zeros(R, f32)
    np.add.at(imp, run, Js)
    np.add.at(nsum, run, dot(Js, nrm))
    cnt = np.bincount(run, minlength=R).astype(np.uint32)
    pen = np.asarray(data["penetration"], f32)
    deepest = np.zeros(R, np.int64)
    depth = np.zeros(R, f32)
    for i in range(n):
        c = srt[i]; r = run[i]
        if head[i]:
            deepest[r] = c; depth[r] = pen[c]
        elif pen[c] > depth[r]:   # strictly deeper: a tie keeps the earlier contact, a NaN never wins
            deepest[r] = c; depth[r] = pen[c]
    out = np.zeros(R, abi.CONTACT_PAIR_IMPULSE)
    out["tags"] = t[head]; out["body_a"] = bodies["a"][deepest]; out["body_b"] = bodies["b"][deepest]
    out["contacts"] = cnt; out["normal_impulse"] = nsum; out["impulse"] = imp; out["penetration"] = pen[deepest]
    return out


def pair_report(data, bodies, tags, impulses, sorted_idx, min_normal_impulse=-np.inf, capacity=None):
    """nb_get_contact_pair_impulses: (the first min(capacity, count) kept rows, count)."""
    rows = pair_rows(data, bodies, tags, impulses, sorted_idx)
    thr = f32(min_normal_impulse)
    if np.isnan(thr):
        raise ValueError("a NaN threshold")
    kept = rows if thr == -np.inf else rows[rows["normal_impulse"] >= thr]
    count = len(kept)
    return (kept if capacity is None else kept[:capacity]), count
