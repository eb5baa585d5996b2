"""CPU restatement of the joint drives with sliders and swing-twist limits (nudge_b200/csrc/nb_joint_api.cuh, k_joint_rows; DESIGN.md sections
8.17 and 8.20) — TEST INFRASTRUCTURE ONLY.

It follows the float32 arithmetic include/nudge_b200.h states for nb_joint_drive, operation by operation, on top of the joints' own rows as
oracle/joints_ref.py builds them.  For drives without SLIDE, CONE and TWIST it gives what tests/joint_drives_ref.py gives (a CPU test holds
the two to the same bytes); the new flags add the slider's rewritten point rows and its motor and limit rows, and BALL's cone and twist
rows.  The device's rows and drive table are compared with it byte for byte; the rows are then solved by the user-row loop
(oracle/rows_ref.py)."""
import numpy as np
from nudge_b200 import ROW
from oracle.joints_ref import ROWS_PER_TYPE, BALL, HINGE, FIXED, DISTANCE, ZERO, f, _v, add, sub, dot, neg, scale, cross, qrot, qmul, \
    joint_rows as own_rows
from tests.joint_drives_ref import LIMIT, MOTOR, BREAKABLE, half_angle, angle_limit_biases

SLIDE, CONE, TWIST = 16, 32, 64
# the device table of nb_debug_read("joint_drives"): one entry per joint (flags 0: none); a CONE drive's (sc, cc) sit in the motor slots
DRIVE_TABLE = np.dtype([("flags", "<u4"), ("row", "<u4"), ("lower", "<f4"), ("upper", "<f4"), ("sl", "<f4"), ("cl", "<f4"), ("su", "<f4"), ("cu", "<f4"),
                        ("motor_speed", "<f4"), ("max_motor_torque", "<f4"), ("break_force", "<f4"), ("break_torque", "<f4"), ("position", "<f4", 2),
                        ("broken", "<u4"), ("cone", "<f4")])
assert DRIVE_TABLE.itemsize == 64
FIRST, RANGE = MOTOR | CONE, LIMIT | TWIST   # the flags that own the first appended row, and the two range rows


def drive_row_count(flags):
    return (1 if flags & FIRST else 0) + (2 if flags & RANGE else 0)


def drive_table(joints, drives):
    """The drive table for `joints` in the order given, from `drives` (nudge_b200.JOINT_DRIVE, joint = an index into `joints`), and the
    appended rows' impulses in row order."""
    table = np.zeros(len(joints), DRIVE_TABLE)
    by = {int(d["joint"]): d for d in drives}
    row, imp = 0, []
    for i, j in enumerate(joints):
        if i not in by:
            continue
        d, e = by[i], table[i]
        fl = int(d["flags"])
        e["flags"], e["row"], e["lower"], e["upper"] = fl, row, d["lower"], d["upper"]
        if (fl & LIMIT and int(j["type"]) == HINGE) or fl & TWIST:
            (e["sl"], e["cl"]), (e["su"], e["cu"]) = half_angle(d["lower"]), half_angle(d["upper"])
        for k in ("motor_speed", "max_motor_torque", "break_force", "break_torque", "broken"):
            e[k] = d[k]
        if fl & CONE:
            (e["motor_speed"], e["max_motor_torque"]), e["cone"] = half_angle(d["cone"]), d["cone"]
        for k in range(3):
            if fl & (RANGE if k else FIRST):
                imp.append(d["impulse"][k])
        row += drive_row_count(fl)
    return table, np.array(imp, np.float32)


def solve_order(joints, table):
    """The permutation of joint_rows' output into solve order: each joint's own rows, then its appended rows."""
    own = np.cumsum([0] + [ROWS_PER_TYPE[int(j["type"])] for j in joints])
    out, extra = [], own[-1]
    for i, j in enumerate(joints):
        out.extend(range(own[i], own[i + 1]))
        c = drive_row_count(int(table["flags"][i]))
        out.extend(range(extra, extra + c)); extra += c
    return np.array(out, np.int64)


def broken_after(joints, rows, table, dt):
    """The break rule: the broken flags after k_joint_rows' test on `rows`, the previous rows as joint_rows lays them out.  A distance
    joint's and a slider's appended rows are linear, every other joint's angular."""
    out = table["broken"].copy()
    n, extra = 0, sum(ROWS_PER_TYPE[int(j["type"])] for j in joints)
    with np.errstate(all="ignore"):
        for i, j in enumerate(joints):
            typ, fl = int(j["type"]), int(table["flags"][i])
            own, c = ROWS_PER_TYPE[typ], drive_row_count(fl)
            if not out[i] and fl & BREAKABLE:
                P = A = f(0.0)
                for r in range(own):
                    x = rows["impulse"][n + r]
                    if typ == DISTANCE or r < 3:
                        P = P + x * x
                    else:
                        A = A + x * x
                for r in range(c):
                    x = rows["impulse"][extra + r]
                    if typ == DISTANCE or fl & SLIDE:
                        P = P + x * x
                    else:
                        A = A + x * x
                lf, lt = table["break_force"][i] * f(dt), table["break_torque"][i] * f(dt)
                if P > lf * lf or A > lt * lt:
                    out[i] = 1
            n += own; extra += c
    return out


def hinge_basis(u):
    """The two unit vectors HINGE builds perpendicular to its axis u."""
    z, o = f(0.0), f(1.0)
    t1 = (z, u[2], -u[1]) if np.abs(u[0]) < f(0.57735) else (-u[2], z, u[0])
    t1 = scale(t1, o / np.sqrt(dot(t1, t1)))
    return t1, cross(u, t1)


def relative(j, transforms):
    """qmul(q_a, rel_rotation), times conj(q_b) when b != 0, with all four components negated when w < 0."""
    a, b = int(j["a"]), int(j["b"])
    q = qmul(_v(transforms["rotation"][a]), _v(j["rel_rotation"]))
    if b:
        qb = _v(transforms["rotation"][b])
        q = qmul(q, neg(qb[:3]) + (qb[3],))
    return tuple(-x for x in q) if q[3] < 0 else q


def swing_twist(q, u):
    """The split of the relative rotation q (w >= 0) about the twist axis u: the swing vector p, (ss, cs) = (sin, cos) of half the swing
    angle, and the twist's half-angle pair (sh', ch')."""
    a_ = dot(q[:3], u)
    sh, ch = -a_, q[3]
    p = sub(q[:3], scale(u, a_))
    ss, cs = np.sqrt(dot(p, p)), np.sqrt(sh * sh + ch * ch)
    if cs > 0:
        r = f(1.0) / cs
        st, ct = sh * r, ch * r
    else:
        st, ct = f(0.0), f(1.0)
    return p, ss, cs, st, ct


def joint_rows(joints, transforms, dt, drives=None, drive_impulse=None):
    """The rows of `joints` (nudge_b200.JOINT) in joint order as oracle/joints_ref.joint_rows builds them; with `drives` (DRIVE_TABLE, one
    entry per joint in the same order) a slider's point rows rewritten, and the drives' rows after all joints' own rows, per driven joint in
    order, with impulses from `drive_impulse` (row order; default 0).  A broken entry's rows are zero rows, and each unbroken entry's
    position is written in place."""
    own = own_rows(joints, transforms, dt)
    if drives is None:
        return own
    n_own = len(own)
    out = np.zeros(n_own + sum(drive_row_count(int(x)) for x in drives["flags"]), ROW)
    out[:n_own] = own
    n, m = 0, n_own
    z, inf = f(0.0), f(np.inf)
    with np.errstate(all="ignore"):
        for i, j in enumerate(joints):
            a, b, typ = int(j["a"]), int(j["b"]), int(j["type"])
            e, fl, count = drives[i], int(drives["flags"][i]), ROWS_PER_TYPE[typ]
            extra = []   # (lin_a, ang_a, lin_b, ang_b, bias, lo, hi)
            if e["broken"]:
                out[n:n + count] = 0; out["a"][n:n + count], out["b"][n:n + count] = a, b
                for r in range(drive_row_count(fl)):
                    out[m]["a"], out[m]["b"] = a, b; m += 1
                n += count
                continue
            k = f(j["beta"]) / f(dt)

            def limit_bias(C):
                return C / f(dt) if C > 0 else k * C
            qa = _v(transforms["rotation"][a])
            ra = qrot(qa, _v(j["anchor_a"]))
            wa = add(_v(transforms["position"][a]), ra)
            rb = qrot(_v(transforms["rotation"][b]), _v(j["anchor_b"])) if b else ZERO
            wb = add(_v(transforms["position"][b]), rb) if b else _v(j["anchor_b"])
            err = sub(wa, wb)
            if typ == DISTANCE and fl & LIMIT:
                r = out[n]
                r["lo"] = r["hi"] = z   # the own row stays in place with no force
                dist = np.sqrt(dot(err, err))
                la, aa, lb, ab = (tuple(r[x]) for x in ("lin_a", "ang_a", "lin_b", "ang_b"))
                extra.append((la, aa, lb, ab, limit_bias(dist - e["lower"]), z, inf))
                extra.append((neg(la), neg(aa), neg(lb), neg(ab), limit_bias(e["upper"] - dist), z, inf))
                e["position"][0] = dist
            if typ == HINGE:
                u = qrot(qa, _v(j["axis_a"]))
                nu = neg(u)
                if fl & MOTOR:
                    lim = e["max_motor_torque"] * f(dt)
                    extra.append((ZERO, nu, ZERO, u, -e["motor_speed"], -lim, lim))
                if fl & LIMIT:
                    q = relative(j, transforms)
                    sh, ch = -dot(q[:3], u), q[3]
                    lo_bias, hi_bias = angle_limit_biases(sh, ch, e, limit_bias)
                    extra.append((ZERO, nu, ZERO, u, lo_bias, z, inf))
                    extra.append((ZERO, u, ZERO, nu, hi_bias, z, inf))
                    e["position"][0], e["position"][1] = sh, ch
            if typ == FIXED and fl & SLIDE:
                u = qrot(qa, _v(j["axis_a"]))
                sa = sub(ra, err)
                t1, t2 = hinge_basis(u)
                for r, t, lo, hi in ((out[n], t1, -inf, inf), (out[n + 1], t2, -inf, inf), (out[n + 2], u, z, z)):
                    r["lin_a"], r["ang_a"], r["lin_b"], r["ang_b"] = t, cross(sa, t), neg(t), neg(cross(rb, t))
                    r["bias"], r["lo"], r["hi"] = k * dot(err, t), lo, hi
                s = dot(sub(wb, wa), u)
                js = (neg(u), neg(cross(sa, u)), u, cross(rb, u))
                if fl & MOTOR:
                    lim = e["max_motor_torque"] * f(dt)
                    extra.append(js + (-e["motor_speed"], -lim, lim))
                if fl & LIMIT:
                    extra.append(js + (limit_bias(s - e["lower"]), z, inf))
                    extra.append(tuple(neg(x) for x in js) + (limit_bias(e["upper"] - s), z, inf))
                e["position"][0] = s
            if typ == BALL and fl & (CONE | TWIST):
                u = qrot(qa, _v(j["axis_a"]))
                q = relative(j, transforms)
                p, ss, cs, st, ct = swing_twist(q, u)
                if fl & CONE:
                    c = cross(qrot(neg(q[:3]) + (q[3],), u), u)
                    sc = np.sqrt(dot(c, c))
                    nv = scale(c, f(1.0) / sc) if sc > 0 else ZERO
                    extra.append((ZERO, neg(nv), ZERO, nv, limit_bias(f(2.0) * (e["motor_speed"] * cs - e["max_motor_torque"] * ss)), z, inf))
                if fl & TWIST:
                    nu = neg(u)
                    lo_bias, hi_bias = angle_limit_biases(st, ct, e, limit_bias)
                    extra.append((ZERO, nu, ZERO, u, lo_bias, z, inf))
                    extra.append((ZERO, u, ZERO, nu, hi_bias, z, inf))
                e["position"][0], e["position"][1] = (st, ct) if fl & TWIST else (ss, cs)
            for la, aa, lb, ab, bias, lo, hi in extra:
                r = out[m]
                r["a"], r["b"] = a, b
                r["lin_a"], r["ang_a"], r["lin_b"], r["ang_b"], r["bias"], r["lo"], r["hi"] = la, aa, lb, ab, bias, lo, hi
                r["impulse"], r["softness"] = (drive_impulse[m - n_own] if drive_impulse is not None else 0.0), j["softness"]
                m += 1
            n += count
    return out


def drive_position(typ, flags, position):
    """The position nb_download_joint_drives reports from a table entry's recorded pair."""
    if typ in (HINGE, BALL) and flags & (LIMIT | CONE | TWIST):
        return f(2.0 * np.arctan2(np.float64(position[0]), np.float64(position[1])))
    return position[0] if flags & (LIMIT | SLIDE) else f(0.0)
