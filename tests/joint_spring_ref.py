"""CPU restatement of the joint springs (nudge_b200/csrc/nb_joint_api.cuh, k_joint_rows; DESIGN.md section 8.21) — TEST INFRASTRUCTURE ONLY.

It follows the float32 arithmetic include/nudge_b200.h states for nb_joint_spring, operation by operation, on top of the joints' own rows and
the drives' rows as tests/joint_dof_ref.py builds them.  Without springs it gives what joint_dof_ref gives.  The device's spring table and
spring rows are compared with it byte for byte; the rows are then solved by the user-row loop (oracle/rows_ref.py) in solve order: per
joint its own rows, its spring rows, its drive rows."""
import numpy as np
from oracle.joints_ref import ROWS_PER_TYPE, BALL, HINGE, FIXED, DISTANCE, ZERO, f, _v, add, sub, dot, neg, cross, qrot, qmul
from tests import joint_dof_ref as dof
from tests.joint_drives_ref import half_angle, angle_limit_measure

# the device table of nb_debug_read("joint_springs"): one entry per joint (present 0: none); a HINGE holds (st, ct) in target[0:2]
SPRING_TABLE = np.dtype([("present", "<u4"), ("row", "<u4"), ("target", "<f4", 4), ("target_velocity", "<f4"), ("stiffness", "<f4"),
                         ("damping", "<f4"), ("max_force", "<f4"), ("position", "<f4", 2), ("angle", "<f4"), ("reserved", "<u4", 3)])
assert SPRING_TABLE.itemsize == 64


def spring_row_count(typ):
    return 3 if typ == BALL else 1


def spring_table(joints, springs):
    """The spring table for `joints` in the order given, from `springs` (nudge_b200.JOINT_SPRING, joint = an index into `joints`), and the
    spring rows' impulses in row order."""
    table = np.zeros(len(joints), SPRING_TABLE)
    by = {int(s["joint"]): s for s in springs}
    row, imp = 0, []
    for i, j in enumerate(joints):
        if i not in by:
            continue
        s, e, typ = by[i], table[i], int(j["type"])
        e["present"], e["row"], e["target"] = 1, row, s["target"]
        if typ == HINGE:
            (e["target"][0], e["target"][1]), e["angle"] = half_angle(s["target"][0]), s["target"][0]
        for k in ("target_velocity", "stiffness", "damping", "max_force"):
            e[k] = s[k]
        imp.extend(s["impulse"][:spring_row_count(typ)])
        row += spring_row_count(typ)
    return table, np.array(imp, np.float32)


def spring_row(r, a, b, la, aa, lb, ab, C, e, dt):
    """The spring row on coordinate C: softness 1 / (dt * den), bias (k * C - c * v_t) / den with den = c + dt * k."""
    dt = f(dt)
    den = e["damping"] + dt * e["stiffness"]
    lim = e["max_force"] * dt
    r["a"], r["b"] = a, b
    r["lin_a"], r["ang_a"], r["lin_b"], r["ang_b"] = la, aa, lb, ab
    r["bias"] = (e["stiffness"] * C - e["damping"] * e["target_velocity"]) / den
    r["lo"], r["hi"], r["softness"], r["reserved"] = -lim, lim, f(1.0) / (dt * den), 0.0


def joint_rows(joints, transforms, dt, drives=None, drive_impulse=None, springs=None, spring_impulse=None):
    """(rows, spring rows): joint_dof_ref.joint_rows' rows for `joints` with `drives`, and with `springs` (SPRING_TABLE, one entry per joint
    in the same order) the spring rows per sprung joint in order, impulses from `spring_impulse` (row order; default 0); a sprung distance
    joint's own row gets lo = hi = 0.  A joint broken in `drives` has zero spring rows; each unbroken spring's position is written in place."""
    rows = dof.joint_rows(joints, transforms, dt, drives, drive_impulse)
    if springs is None:
        return rows, np.zeros(0, rows.dtype)
    out = np.zeros(sum(spring_row_count(int(j["type"])) for j, e in zip(joints, springs) if e["present"]), rows.dtype)
    n, m = 0, 0
    z = f(0.0)
    with np.errstate(all="ignore"):
        for i, j in enumerate(joints):
            a, b, typ = int(j["a"]), int(j["b"]), int(j["type"])
            count, e = ROWS_PER_TYPE[typ], springs[i]
            if not e["present"]:
                n += count
                continue
            c = spring_row_count(typ)
            out["impulse"][m:m + c] = spring_impulse[m:m + c] if spring_impulse is not None else 0.0
            if drives is not None and drives["broken"][i]:
                out[m:m + c] = 0; out["a"][m:m + c], out["b"][m:m + c] = a, b
                n += count; m += c
                continue
            qa = _v(transforms["rotation"][a])
            ra = qrot(qa, _v(j["anchor_a"]))
            wa = add(_v(transforms["position"][a]), ra)
            rb = qrot(_v(transforms["rotation"][b]), _v(j["anchor_b"])) if b else ZERO
            wb = add(_v(transforms["position"][b]), rb) if b else _v(j["anchor_b"])
            err = sub(wa, wb)
            if typ == DISTANCE:
                own = rows[n]
                own["lo"] = own["hi"] = z
                dist = np.sqrt(dot(err, err))
                spring_row(out[m], a, b, *(tuple(own[x]) for x in ("lin_a", "ang_a", "lin_b", "ang_b")), dist - e["target"][0], e, dt)
                e["position"][0] = dist
            elif typ == HINGE:
                u = qrot(qa, _v(j["axis_a"]))
                q = dof.relative(j, transforms)
                sh, ch = -dot(q[:3], u), q[3]
                st, ct = e["target"][0], e["target"][1]
                spring_row(out[m], a, b, ZERO, neg(u), ZERO, u, angle_limit_measure(sh * ct - ch * st, ch * ct + sh * st), e, dt)
                e["position"][0], e["position"][1] = sh, ch
            elif typ == FIXED:
                u = qrot(qa, _v(j["axis_a"]))
                sa = sub(ra, err)
                s = dot(sub(wb, wa), u)
                spring_row(out[m], a, b, neg(u), neg(cross(sa, u)), u, cross(rb, u), s - e["target"][0], e, dt)
                e["position"][0] = s
            else:
                q = qmul(qa, _v(e["target"]))
                if b:
                    qb = _v(transforms["rotation"][b])
                    q = qmul(q, neg(qb[:3]) + (qb[3],))
                if q[3] < 0:
                    q = tuple(-x for x in q)
                for k in range(3):   # ang_a = e, ang_b = -e with +0 in the other components, as FIXED's rows
                    e_, ne = (tuple(f(v) if x == k else z for x in range(3)) for v in (1.0, -1.0))
                    spring_row(out[m + k], a, b, ZERO, e_, ZERO, ne, f(2.0) * q[k], e, dt)
                e["position"][0], e["position"][1] = np.sqrt(dot(q[:3], q[:3])), q[3]
            n += count; m += c
    return rows, out


def solve_order(joints, drives, springs):
    """The permutation of concatenate((rows, spring rows)) into solve order: per joint its own rows, its spring rows, its drive rows."""
    own = np.cumsum([0] + [ROWS_PER_TYPE[int(j["type"])] for j in joints])
    flags = drives["flags"] if drives is not None else np.zeros(len(joints), np.uint32)
    n_rows = own[-1] + sum(dof.drive_row_count(int(x)) for x in flags)
    out, extra, spring = [], own[-1], n_rows
    for i, j in enumerate(joints):
        out.extend(range(own[i], own[i + 1]))
        if springs is not None and springs["present"][i]:
            c = spring_row_count(int(j["type"]))
            out.extend(range(spring, spring + c)); spring += c
        c = dof.drive_row_count(int(flags[i]))
        out.extend(range(extra, extra + c)); extra += c
    return np.array(out, np.int64)


def spring_position(typ, position):
    """The position nb_download_joint_springs reports from a table entry's recorded pair."""
    if typ in (HINGE, BALL):
        return f(2.0 * np.arctan2(np.float64(position[0]), np.float64(position[1])))
    return position[0]
