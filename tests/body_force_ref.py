"""Restatement of the force stage with a per-body force table (nb_set_body_forces; include/nudge_b200.h, DESIGN.md section 8.11) in numpy
float32, with the header's operation order (left to right, no fused multiply-add), and an OracleSim whose apply_gravity_damping is that
stage.  The table is held as B BODY_FORCE rows (body = the row index), as nb_download_body_forces returns it."""
import numpy as np
from nudge_b200 import scenes
from oracle import pyoracle
from tests.impulse_ref import world_inverse_inertia
from tests.spawn_ref import body_map

F = np.float32


def default_table(n_bodies):
    return scenes.default_body_forces(np.arange(n_bodies))


def set_entries(table, rows):
    """nb_set_body_forces on a table: the listed entries replace their bodies' rows (reserved stored as 0)."""
    rows = np.asarray(rows, scenes.BODY_FORCE).reshape(-1)
    table[rows["body"].astype(np.int64)] = rows
    table["reserved"] = 0


def _cross(a, b):
    return np.stack([a[:, 1] * b[:, 2] - a[:, 2] * b[:, 1], a[:, 2] * b[:, 0] - a[:, 0] * b[:, 2], a[:, 0] * b[:, 1] - a[:, 1] * b[:, 0]], 1)


def qrot(q, r):
    """nb_common.cuh qrot (nudge.cpp:1117-1120) row by row: t = 2 * cross(q.xyz, r); (r + q.w * t) + cross(q.xyz, t).  q (n, 4) x, y, z, w."""
    q = np.asarray(q, F).reshape(-1, 4); r = np.asarray(r, F).reshape(-1, 3)
    v, s = q[:, :3], q[:, 3:4]
    t = F(2.0) * _cross(v, r)
    return ((r + s * t) + _cross(v, t)).astype(F)


def apply_stage(state, table, active, time_step, gravity, damping, kinematic=()):
    """The force stage on the host arrays of `state` (momentum, idle, transforms, properties) for the body indices `active`, kinematic bodies
    skipped.  Returns the bodies that carried a force or torque (their idle counters are now 0)."""
    dt, g, d = F(time_step), F(gravity), F(damping)
    kin = set(int(k) for k in kinematic)
    idx = np.array([i for i in np.asarray(active).tolist() if i not in kin], np.int64)
    if not len(idx):
        return idx
    e = table[idx]
    m = state.momentum
    v = m["velocity"][idx].astype(F)
    w = m["angular_velocity"][idx].astype(F)
    dv = g * dt
    v[:, 1] = v[:, 1] - dv * e["gravity_scale"].astype(F)
    f, t = e["force"].astype(F), e["torque"].astype(F)
    hf, ht = (f != 0).any(1), (t != 0).any(1)   # -0.0 == 0
    local = (e["flags"] & scenes.BODY_FORCE_LOCAL) != 0
    q = state.transforms["rotation"][idx].astype(F)
    with np.errstate(all="ignore"):
        f = np.where(local[:, None], qrot(q, f), f)
        t = np.where(local[:, None], qrot(q, t), t)
        k = state.properties["mass_inverse"][idx].astype(F) * dt
        for c in range(3):
            v[hf, c] = v[hf, c] + f[hf, c] * k[hf]
        W = world_inverse_inertia(q, state.properties[idx])
        xx, yy, zz, xy, xz, yz = (W[:, j] for j in range(6))
        tx, ty, tz = t[:, 0], t[:, 1], t[:, 2]
        w[ht, 0] = w[ht, 0] + (((xx * tx + xy * ty) + xz * tz) * dt)[ht]
        w[ht, 1] = w[ht, 1] + (((xy * tx + yy * ty) + yz * tz) * dt)[ht]
        w[ht, 2] = w[ht, 2] + (((xz * tx + yz * ty) + zz * tz) * dt)[ht]
    lin = F(1.0) - dt * (d + e["linear_damping"].astype(F))
    ang = F(1.0) - dt * (d + e["angular_damping"].astype(F))
    m["velocity"][idx] = v * lin[:, None]
    m["angular_velocity"][idx] = w * ang[:, None]
    pushed = idx[hf | ht]
    state.idle[pushed] = 0
    return pushed


def remove_table(table, idx):
    """nb_remove_bodies on the table: the kept rows in order, each renamed to its body's new index."""
    keep, m = body_map(len(table), idx)
    out = table[keep].copy()
    out["body"] = m[keep]
    return out


def add_table(table, n):
    """nb_add_bodies on the table: n default rows appended."""
    return np.concatenate([table, scenes.default_body_forces(np.arange(len(table), len(table) + n))])


class BodyForceOracleSim(pyoracle.OracleSim):
    """OracleSim with a body force table (Scene.body_forces or set_body_forces); without a table its step is the oracle's."""

    def __init__(self, scene, ftz=False, contact_capacity=None):
        super().__init__(scene, ftz, contact_capacity)
        self.table = None
        if getattr(scene, "body_forces", None) is not None:
            self.set_body_forces(scene.body_forces)

    def set_body_forces(self, rows):
        if self.table is None:
            self.table = default_table(self.scene.n_bodies)
        rows = np.asarray(rows, scenes.BODY_FORCE).reshape(-1)
        set_entries(self.table, rows)
        self.idle[rows["body"].astype(np.int64)] = 0

    def clear_body_forces(self):
        self.table = None

    def apply_gravity_damping(self):
        if self.table is None:
            return super().apply_gravity_damping()
        s = self.scene
        apply_stage(self, self.table, self.active_indices[:self.active.count], s.time_step, s.gravity, s.damping)
