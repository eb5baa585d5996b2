"""CPU restatement of the joint drives (nudge_b200/csrc/nb_joint_api.cuh, k_joint_rows; DESIGN.md section 8.17) — TEST INFRASTRUCTURE ONLY.

It follows the float32 arithmetic include/nudge_b200.h states for nb_joint_drive, operation by operation, on top of the joints' own rows as
oracle/joints_ref.py builds them, so the device's rows and drive table are compared with it byte for byte; the rows are then solved by the
user-row loop (oracle/rows_ref.py)."""
import numpy as np
from nudge_b200 import ROW
from oracle.joints_ref import ROWS_PER_TYPE, HINGE, DISTANCE, ZERO, f, _v, add, sub, dot, neg, qrot, qmul, joint_rows as own_rows

LIMIT, MOTOR, BREAKABLE = 1, 2, 4
# the device table of nb_debug_read("joint_drives"): one entry per joint (flags 0: none)
DRIVE_TABLE = np.dtype([("flags", "<u4"), ("row", "<u4"), ("lower", "<f4"), ("upper", "<f4"), ("sl", "<f4"), ("cl", "<f4"), ("su", "<f4"), ("cu", "<f4"),
                        ("motor_speed", "<f4"), ("max_motor_torque", "<f4"), ("break_force", "<f4"), ("break_torque", "<f4"), ("position", "<f4", 2),
                        ("broken", "<u4"), ("reserved", "<u4")])
assert DRIVE_TABLE.itemsize == 64


def drive_row_count(flags):
    return (1 if flags & MOTOR else 0) + (2 if flags & LIMIT else 0)


def half_angle(x):
    """(sin(x/2), cos(x/2)) of a hinge limit as the upload converts it: in double, rounded to float32."""
    return f(np.sin(0.5 * np.float64(f(x)))), f(np.cos(0.5 * np.float64(f(x))))


def angle_limit_measure(s, c):
    """An angle limit's C from (s, c) = (sin x, cos x) of the half difference x = (angle - stop) / 2: 2 sin x while c >= 0, then
    +-(4 - 2 |sin x|) with the sign of x (float32 add, multiply and compare only)."""
    t = f(2.0) * s
    return t if c >= 0 else (f(4.0) - t if s >= 0 else f(-4.0) - t)


def angle_limit_biases(sh, ch, e, limit_bias):
    """The lower and upper angle limit rows' biases from the angle's half-angle pair (sh, ch) and the entry's limit pairs."""
    return (limit_bias(angle_limit_measure(sh * e["cl"] - ch * e["sl"], ch * e["cl"] + sh * e["sl"])),
            limit_bias(angle_limit_measure(e["su"] * ch - e["cu"] * sh, e["cu"] * ch + e["su"] * sh)))


def drive_table(joints, drives):
    """The drive table for `joints` in the order given, from `drives` (nudge_b200.JOINT_DRIVE, joint = an index into `joints`): the entries of
    nb_upload_joint_drives with the half-angle pairs and each drive's first row in the drive rows; and the appended rows' impulses in row
    order."""
    table = np.zeros(len(joints), DRIVE_TABLE)
    by = {int(d["joint"]): d for d in drives}
    row, imp = 0, []
    for i, j in enumerate(joints):
        if i not in by:
            continue
        d, e = by[i], table[i]
        fl = int(d["flags"])
        e["flags"], e["row"], e["lower"], e["upper"] = fl, row, d["lower"], d["upper"]
        if fl & LIMIT and int(j["type"]) == HINGE:
            (e["sl"], e["cl"]), (e["su"], e["cu"]) = half_angle(d["lower"]), half_angle(d["upper"])
        for k in ("motor_speed", "max_motor_torque", "break_force", "break_torque", "broken"):
            e[k] = d[k]
        for k in range(3):
            if fl & (LIMIT if k else MOTOR):
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
    """The break rule: the broken flags after k_joint_rows' test on `rows`, the previous rows as joint_rows lays them out (their impulses
    are what the previous step left)."""
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
                    if typ == DISTANCE:
                        P = P + x * x
                    else:
                        A = A + x * x
                lf, lt = table["break_force"][i] * f(dt), table["break_torque"][i] * f(dt)
                if P > lf * lf or A > lt * lt:
                    out[i] = 1
            n += own; extra += c
    return out


def joint_rows(joints, transforms, dt, drives=None, drive_impulse=None):
    """The rows of `joints` (nudge_b200.JOINT) in joint order as oracle/joints_ref.joint_rows builds them; with `drives` (DRIVE_TABLE, one
    entry per joint in the same order) the drives' rows follow all joints' own rows, per driven joint in order, with impulses from
    `drive_impulse` (row order; default 0).  A broken entry's rows are zero rows, and each unbroken LIMIT entry's position is written in place."""
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
            if typ == DISTANCE and fl & LIMIT:
                r = out[n]
                r["lo"] = r["hi"] = z   # the own row stays in place with no force
                ra = qrot(qa, _v(j["anchor_a"]))
                wa = add(_v(transforms["position"][a]), ra)
                wb = add(_v(transforms["position"][b]), qrot(_v(transforms["rotation"][b]), _v(j["anchor_b"]))) if b else _v(j["anchor_b"])
                err = sub(wa, wb)
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
                    q = qmul(qa, _v(j["rel_rotation"]))
                    if b:
                        qb = _v(transforms["rotation"][b])
                        q = qmul(q, neg(qb[:3]) + (qb[3],))
                    if q[3] < 0:
                        q = tuple(-x for x in q)
                    sh, ch = -dot(q[:3], u), q[3]
                    lo_bias, hi_bias = angle_limit_biases(sh, ch, e, limit_bias)
                    extra.append((ZERO, nu, ZERO, u, lo_bias, z, inf))
                    extra.append((ZERO, u, ZERO, nu, hi_bias, z, inf))
                    e["position"][0], e["position"][1] = sh, ch
            for la, aa, lb, ab, bias, lo, hi in extra:
                r = out[m]
                r["a"], r["b"] = a, b
                r["lin_a"], r["ang_a"], r["lin_b"], r["ang_b"], r["bias"], r["lo"], r["hi"] = la, aa, lb, ab, bias, lo, hi
                r["impulse"], r["softness"] = (drive_impulse[m - n_own] if drive_impulse is not None else 0.0), j["softness"]
                m += 1
            n += count
    return out
