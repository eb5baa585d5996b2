"""CPU restatement of the joints' row construction (nudge_b200/csrc/nb_joint_api.cuh, k_joint_rows) — TEST INFRASTRUCTURE ONLY.

The reference has no joints.  This follows the float32 arithmetic include/nudge_b200.h states for nb_joint, operation by operation, so the
device's rows are compared with it byte for byte; the rows are then solved by the user-row loop (oracle/rows_ref.py)."""
import numpy as np
from nudge_b200 import ROW

f = np.float32
ROWS_PER_TYPE = (3, 5, 6, 1)   # BALL, HINGE, FIXED, DISTANCE
BALL, HINGE, FIXED, DISTANCE = 0, 1, 2, 3
ZERO = (f(0.0), f(0.0), f(0.0))


def _v(a):
    return tuple(f(x) for x in a)


def cross(u, v):
    return (u[1] * v[2] - u[2] * v[1], u[2] * v[0] - u[0] * v[2], u[0] * v[1] - u[1] * v[0])


def dot(u, v):
    return (u[0] * v[0] + u[1] * v[1]) + u[2] * v[2]


def add(u, v):
    return (u[0] + v[0], u[1] + v[1], u[2] + v[2])


def sub(u, v):
    return (u[0] - v[0], u[1] - v[1], u[2] - v[2])


def scale(u, s):
    return (u[0] * s, u[1] * s, u[2] * s)


def neg(u):
    return (-u[0], -u[1], -u[2])


def qrot(q, r):
    t = scale(cross(q[:3], r), f(2.0))
    return add(add(r, scale(t, q[3])), cross(q[:3], t))


def qmul(l, r):
    v = add(add(scale(r[:3], l[3]), scale(l[:3], r[3])), cross(l[:3], r[:3]))
    return v + (l[3] * r[3] - dot(l[:3], r[:3]),)


def joint_rows(joints, transforms, dt):
    """The rows of `joints` (nudge_b200.JOINT) in joint order from `transforms` (position, rotation per body); impulse = the joints' impulse[]."""
    out = np.zeros(sum(ROWS_PER_TYPE[int(j["type"])] for j in joints), ROW)
    n = 0
    with np.errstate(all="ignore"):
        for j in joints:
            a, b, typ = int(j["a"]), int(j["b"]), int(j["type"])
            k = f(j["beta"]) / f(dt)
            qa = _v(transforms["rotation"][a])
            ra = qrot(qa, _v(j["anchor_a"])); wa = add(_v(transforms["position"][a]), ra)
            rb, wb, qb = ZERO, _v(j["anchor_b"]), None
            if b:
                qb = _v(transforms["rotation"][b])
                rb = qrot(qb, _v(j["anchor_b"])); wb = add(_v(transforms["position"][b]), rb)
            err = sub(wa, wb)
            o, z = f(1.0), f(0.0)
            rows = []   # (lin_a, ang_a, lin_b, ang_b, bias)
            if typ == DISTANCE:
                dist = np.sqrt(dot(err, err))
                d = scale(err, o / dist) if dist > 0 else (z, o, z)
                rows.append((d, cross(ra, d), neg(d), neg(cross(rb, d)), k * (dist - f(j["length"]))))
            else:
                rows.append(((o, z, z), (z, ra[2], -ra[1]), (-o, z, z), (z, -rb[2], rb[1]), k * err[0]))
                rows.append(((z, o, z), (-ra[2], z, ra[0]), (z, -o, z), (rb[2], z, -rb[0]), k * err[1]))
                rows.append(((z, z, o), (ra[1], -ra[0], z), (z, z, -o), (-rb[1], rb[0], z), k * err[2]))
            if typ == HINGE:
                u = qrot(qa, _v(j["axis_a"])); w = qrot(qb, _v(j["axis_b"])) if b else _v(j["axis_b"])
                c = cross(u, w)
                t1 = (z, u[2], -u[1]) if np.abs(u[0]) < f(0.57735) else (-u[2], z, u[0])
                t1 = scale(t1, o / np.sqrt(dot(t1, t1)))
                for t in (t1, cross(u, t1)):
                    rows.append((ZERO, t, ZERO, neg(t), -(k * dot(c, t))))
            if typ == FIXED:
                d = qmul(qa, _v(j["rel_rotation"]))
                if b:
                    d = qmul(d, neg(qb[:3]) + (qb[3],))
                dv = neg(d[:3]) if d[3] < 0 else d[:3]
                for e in range(3):
                    ax = tuple(o if i == e else z for i in range(3)); nx = tuple(-o if i == e else z for i in range(3))
                    rows.append((ZERO, ax, ZERO, nx, k * (f(2.0) * dv[e])))
            for i, (la, aa, lb, ab, bias) in enumerate(rows):
                r = out[n]; n += 1
                r["a"], r["b"] = a, b
                r["lin_a"], r["ang_a"], r["lin_b"], r["ang_b"], r["bias"] = la, aa, lb, ab, bias
                r["lo"], r["hi"], r["impulse"], r["softness"] = -np.inf, np.inf, j["impulse"][i], j["softness"]
    return out


def joint_levels(joints):
    """Each joint's dependency level: 1 + the highest level of an earlier joint on either of its bodies (body 0 is shared freely)."""
    last, levels = {}, []
    for j in joints:
        bodies = [int(x) for x in (j["a"], j["b"]) if int(x)]
        lv = max([last[x] + 1 for x in bodies if x in last], default=0)
        for x in bodies:
            last[x] = lv
        levels.append(lv)
    return np.asarray(levels, np.int64)


def table_order(joints):
    """The joint indices in device table order: by level, upload order within one (the order of nb_debug_read's "joint_rows")."""
    return np.argsort(joint_levels(joints), kind="stable")


def set_impulses(joints, rows):
    """Copies the impulses of `rows` (as joint_rows lays them out) back into joints['impulse']."""
    n = 0
    for j in joints:
        c = ROWS_PER_TYPE[int(j["type"])]
        j["impulse"] = 0
        j["impulse"][:c] = rows["impulse"][n:n + c]; n += c
