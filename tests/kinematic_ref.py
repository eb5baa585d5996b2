"""Test infrastructure: kinematic bodies (include/nudge_b200.h nb_upload_kinematic_bodies) restated on top of the unmodified widened CPU oracle.

A kinematic body is "body 0 with a velocity": the oracle already reads body 0's velocity in the warm start and the sweeps, gives it the inverse
mass and inertia of its properties row, substitutes it in the scheduler and never waits on it.  So for a scene with ONE kinematic body K whose
static world (body 0) carries no collider, every oracle stage runs with K and body 0 swapped (K's properties row zeroed: infinite mass), and
the results are mapped back.  Any other set (several kinematic bodies, or colliders left on body 0) is restated through the collide stage,
gravity and advance, which need no swap; setup and the sweeps refuse it (tests step the device and copy its state in, sync_oracle_from_gpu).  What the oracle cannot know is restated here:
  - the collide stage, by tests/filter_ref.py restate_collide as for the filter: the oracle runs with every body awake (all pairs, every pair's
    contacts in pipeline order), pairs of two non-dynamic bodies with a kinematic one are dropped, and both island passes are redone with the
    kinematic rules: a kinematic body never joins a set, an edge to a MOVING one (any nonzero velocity component) makes the dynamic side's set
    active, an edge to one at rest is ignored; a moving kinematic body is active itself;
  - gravity and damping skip kinematic bodies;
  - a kinematic momentum row is never written: the oracle's setup and sweeps write body 0's row back (unchanged velocities, since its inverse
    mass and inertia are zero, but unused1 = 0), so the row is restored after them, with unused0 = 0 as setup writes it.  Exact for
    velocities without -0.0 components (the oracle's write-back may turn -0.0 into +0.0);
  - nb_advance integrates a moving kinematic body with the oracle's own arithmetic (it is in the active list).
With no set or an empty set the restatement is the oracle's own result, bit for bit (tests/test_kinematic_oracle.py checks this over a run
that sleeps and wakes).  Contacts are matched to pairs by their collider tags, so scenes must give every collider a distinct tag."""
import numpy as np
from nudge_b200 import scenes as S
from oracle import pyoracle
from tests.filter_ref import restate_collide


def moving(momentum, body):
    m = momentum[body]
    return bool(np.any(m["velocity"] != 0) or np.any(m["angular_velocity"] != 0))   # -0.0 == 0


class KinematicOracleSim(pyoracle.OracleSim):
    """OracleSim with kinematic bodies (Scene.kinematic or upload_kinematic_bodies); every array it exposes is in the scene's body indices."""

    def __init__(self, scene, ftz=False, contact_capacity=None):
        super().__init__(scene, ftz, contact_capacity)
        self.kin = []
        self.upload_kinematic_bodies(getattr(scene, "kinematic", None))

    def upload_kinematic_bodies(self, rows):
        """Mirror of Sim.upload_kinematic_bodies: replaces the set, writes the velocities; None or empty removes the set."""
        rows = np.asarray(rows if rows is not None else [], S.KINEMATIC).reshape(-1)
        body = [int(b) for b in rows["body"]]
        assert 0 not in body and len(set(body)) == len(body) and all(b < self.scene.n_bodies for b in body)
        cb = np.concatenate([self.box_transforms["body"], self.sphere_transforms["body"]])
        self.swappable = len(body) == 1 and not (cb == 0).any()   # the solver stages need one kinematic body and a static world without colliders
        for r in rows:
            self.momentum["velocity"][r["body"]] = r["velocity"]
            self.momentum["angular_velocity"][r["body"]] = r["angular_velocity"]
        self.kin = body

    # ---- the swap of K and body 0 around every oracle call ----
    def _swap(self, to_oracle):
        if not self.kin or not self.swappable:
            return
        k = self.kin[0]

        def perm(a):
            a = a.astype(np.int64)
            return np.where(a == k, 0, np.where(a == 0, k, a))
        for arr in (self.transforms, self.properties, self.momentum, self.idle):
            arr[[0, k]] = arr[[k, 0]]
        if to_oracle:
            self._props_k = self.properties[0].copy()
            self.properties[0] = np.zeros(1, S.PROPERTIES)[0]
        else:
            self.properties[k] = self._props_k
        for t in (self.box_transforms, self.sphere_transforms):
            t["body"] = perm(t["body"])
        if len(self.connections):
            self.connections["a"] = perm(self.connections["a"]); self.connections["b"] = perm(self.connections["b"])
        n = self.contacts.count
        self.contact_bodies["a"][:n] = perm(self.contact_bodies["a"][:n]); self.contact_bodies["b"][:n] = perm(self.contact_bodies["b"][:n])
        m = self.active.count
        self.active_indices[:m] = perm(self.active_indices[:m])

    def _oracle(self, f):
        self._swap(True)
        try:
            f()
        finally:
            self._swap(False)

    def _keep_kinematic_rows(self, row):
        for k in self.kin:
            self.momentum[k] = row[k]

    # ---- stages ----
    def collide(self):
        kin = set(self.kin)
        nondyn = kin | {0}

        def keep(body, lo, hi):   # pairs of two non-dynamic bodies, one of them kinematic, are not broadphase pairs
            return np.array([not (a in nondyn and b in nondyn and (a in kin or b in kin)) for a, b in zip(body[lo].tolist(), body[hi].tolist())], bool)
        oracle_collide = super().collide
        restate_collide(self, lambda: self._oracle(oracle_collide), keep, kin, set(k for k in self.kin if moving(self.momentum, k)))

    def pairs_view(self):
        return dict(self._pairs)

    def apply_gravity_damping(self):
        f = np.float32
        dt = f(self.scene.time_step)
        damping = f(f(1.0) - dt * f(self.scene.damping))
        idx = np.array([i for i in self.active_indices[:self.active.count].tolist() if i not in self.kin], np.int64)
        m = self.momentum
        m["velocity"][idx, 1] = m["velocity"][idx, 1] - f(f(self.scene.gravity) * dt)
        m["velocity"][idx] = m["velocity"][idx] * damping
        m["angular_velocity"][idx] = m["angular_velocity"][idx] * damping

    def read_cached_impulses(self):
        self._oracle(super().read_cached_impulses)

    def _solver_ok(self):
        assert not self.kin or self.swappable, "the solver stages are restated for one kinematic body and a static world without colliders"

    def setup_contact_constraints(self):
        self._solver_ok()
        row = self.momentum.copy()
        for k in self.kin:
            row[k]["unused0"] = 0.0
        self._kin_rows = row
        self._oracle(super().setup_contact_constraints)
        self._keep_kinematic_rows(row)

    def apply_impulses(self):
        self._solver_ok()
        self._oracle(super().apply_impulses)
        self._keep_kinematic_rows(self._kin_rows)

    def advance(self):
        self._oracle(super().advance)

    def constraints_view(self):
        """Row bodies in the scene's indices, a kinematic side marked with READ_ONLY as the device's row_a / row_b carry it."""
        v = super().constraints_view()
        if self.kin and self.swappable:
            k = self.kin[0]
            for f in ("a", "b"):
                x = v[f].astype(np.int64)
                v[f] = np.where(x == 0, k | READ_ONLY, np.where(x == k, 0, x)).astype(np.uint32)
        return v


READ_ONLY = 0x80000000   # NB_READ_ONLY of nb_solver.cuh


def with_kinematic_ground(scene, rows_velocity=(0.0, 0.0, 0.0), angular_velocity=(0.0, 0.0, 0.0)):
    """The scene with one extra body K = n_bodies (identity pose, the static world's properties and momentum) carrying every collider of
    body 0 (same tags, same local transforms), kinematic at the given velocity.  Returns (scene, K)."""
    s = scene.copy()
    k = s.n_bodies
    s.transforms = np.concatenate([s.transforms, s.transforms[:1]])
    s.properties = np.concatenate([s.properties, s.properties[:1]])
    s.momentum = np.concatenate([s.momentum, s.momentum[:1]])
    s.idle = np.concatenate([s.idle, s.idle[:1]])
    for t in (s.box_transforms, s.sphere_transforms):
        t["body"][t["body"] == 0] = k
    s.kinematic = np.zeros(1, S.KINEMATIC)
    s.kinematic["body"] = k; s.kinematic["velocity"] = rows_velocity; s.kinematic["angular_velocity"] = angular_velocity
    return s, k


class AsGround:
    """Views a KinematicOracleSim of with_kinematic_ground(scene) in the original scene's body indices (K -> 0, body 0 dropped), for
    tests/parity_util.ref_layout_stages: every stage then compares with the unmodified reference on the original scene."""

    def __init__(self, sim, k):
        self._sim, self._k = sim, k
        self._rows = np.array([k] + list(range(1, k)), np.int64)

    def __getattr__(self, name):
        return getattr(self._sim, name)

    @property
    def momentum(self):
        return self._sim.momentum[self._rows]

    @property
    def transforms(self):
        return self._sim.transforms[self._rows]

    @property
    def idle(self):
        return self._sim.idle[self._rows]

    def contacts_view(self):
        c = self._sim.contacts_view()
        for f in ("a", "b"):
            c["bodies"][f][c["bodies"][f] == self._k] = 0
        return c


def two_kinematic_platforms(n=300, seed=4):
    """A box pile on two kinematic slabs K1 = n + 1 (x < 0) and K2 = n + 2 (x > 0) that overlap each other and the ground, which stays on body 0;
    the lowest layer of boxes already rests on the slabs.  Both kinematic at rest (Scene.kinematic).  Returns (scene, K1, K2)."""
    s = S.box_drop(n, iterations=4, seed=seed, density_L=10.0, spacing=(2.2, 2.2, 2.2), rotate=False)
    y = s.transforms["position"][1:, 1]
    s.transforms["position"][1:, 1] = y - (y.min() - 1.0)
    k1, k2 = s.n_bodies, s.n_bodies + 1
    s.transforms = np.concatenate([s.transforms, s.transforms[:1], s.transforms[:1]])
    s.properties = np.concatenate([s.properties, s.properties[1:3]])   # a dynamic body's properties: a kinematic body ignores them
    s.momentum = np.concatenate([s.momentum, s.momentum[:2]])
    s.idle = np.concatenate([s.idle, s.idle[:2]])
    nb = s.n_boxes
    s.box_tags = np.concatenate([s.box_tags, np.array([nb, nb + 1], np.uint32)])
    s.box_data = np.concatenate([s.box_data, s.box_data[:2]])
    s.box_data["size"][nb:] = (5.6, 0.5, 12.0)
    s.box_transforms = np.concatenate([s.box_transforms, s.box_transforms[:2]])
    s.box_transforms["position"][nb] = (-5.5, 0.4, 0.0); s.box_transforms["body"][nb] = k1
    s.box_transforms["position"][nb + 1] = (5.5, 0.4, 0.0); s.box_transforms["body"][nb + 1] = k2
    s.kinematic = np.zeros(2, S.KINEMATIC); s.kinematic["body"] = (k1, k2)
    return s, k1, k2
