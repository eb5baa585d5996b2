"""Test infrastructure: sensor colliders (include/nudge_b200.h nb_upload_sensors, DESIGN.md section 8.7) restated on top of the filtered
restatement of the CPU oracle (tests/filter_ref.py).

  - Physics: a pair with a sensor in it never becomes a broadphase pair (a sensor pair goes to the sensor list, a pair of two sensors and a
    sensor with a collider of its own body go nowhere), so the physics is FilteredOracleSim with every pair that involves a sensor collider
    rejected, which is what category 0 and mask 0 on the sensor colliders do.
  - Overlaps: FilteredOracleSim.collide first runs the unmodified oracle with every body awake, which gives every pair and its contacts in
    the pipeline's own orientation (kept as awake_pairs and awake_tags).  A sensor pair (exactly one sensor, different bodies, passing the user's filter and connected opt-out)
    overlaps iff it has at least one of those contacts.  Entry: tags = min | max << 32 of the collider tags, body_a = the body of the
    lower-tag collider; the list is sorted by tags.
  - Events: write_cached_impulses diffs the step's overlaps against those of its previous call, like the device.
Contacts are matched to pairs by their collider tags, so scenes must give every collider a distinct tag."""
import numpy as np
from nudge_b200 import scenes
from tests.filter_ref import FilteredOracleSim, pair_passes


def overlap_events(old, cur, step):
    """Sensor events of one write_cached_impulses: ENDs (old keys not in cur) then BEGINs (cur keys not in old), each ascending by key."""
    ends = old[~np.isin(old["tags"], cur["tags"])]
    begins = cur[~np.isin(cur["tags"], old["tags"])]
    out = np.zeros(len(ends) + len(begins), scenes.CONTACT_EVENT)
    for k, (part, kind) in enumerate(((ends, scenes.SENSOR_END), (begins, scenes.SENSOR_BEGIN))):
        sl = slice(0, len(ends)) if k == 0 else slice(len(ends), len(out))
        out["tags"][sl] = part["tags"]; out["kind"][sl] = kind; out["body_a"][sl] = part["body_a"]; out["body_b"][sl] = part["body_b"]
    out["step"] = step
    return out


class SensorOracleSim(FilteredOracleSim):
    """FilteredOracleSim with the scene's (or the uploaded) sensor table: physics without the sensor pairs, plus the overlap list of every
    collide (self.overlaps) and the sensor events of every write_cached_impulses (self.sensor_events(step))."""

    def __init__(self, scene, ftz=False, contact_capacity=None):
        self.sensors = None
        self.user_filters, self.filter_flags = None, 0
        super().__init__(scene, ftz, contact_capacity)
        self.upload_sensors(getattr(scene, "sensors", None))

    def upload_collision_filters(self, filters, flags=0):
        self.user_filters = None if filters is None or len(filters) == 0 else np.array(filters, copy=True)
        self.filter_flags = int(flags)
        self._combine()

    def upload_sensors(self, flags):
        """Mirror of Sim.upload_sensors: None (or empty) removes the table; the old overlap list is emptied either way."""
        self.sensors = None if flags is None or len(flags) == 0 else np.asarray(flags) != 0
        self._combine()
        self.overlaps = np.zeros(0, scenes.SENSOR_OVERLAP)
        self.old = np.zeros(0, scenes.SENSOR_OVERLAP)
        self._diff = (self.old, self.old)

    def _combine(self):
        """The table the physics uses: the user's filters, with category 0 and mask 0 on every sensor collider."""
        f = self.user_filters
        if self.sensors is not None and self.sensors.any():
            if f is None:
                f = np.zeros(len(self.sensors), scenes.FILTER); f["category"] = 0xffff; f["mask"] = 0xffff
            f = f.copy()
            f["category"][self.sensors] = 0; f["mask"][self.sensors] = 0
        self.filters = f

    def collide(self):
        super().collide()
        self.overlaps = self._overlaps()

    def _overlaps(self):
        out = np.zeros(0, scenes.SENSOR_OVERLAP)
        if self.sensors is None:
            return out
        v = self.awake_pairs
        lo, hi = v["lo"].astype(np.int64), v["hi"].astype(np.int64)
        body = np.concatenate([self.box_transforms["body"], self.sphere_transforms["body"]]).astype(np.int64)
        tag = np.concatenate([self.box_tags, self.sphere_tags]).astype(np.uint64)
        connected = set((min(int(c["a"]), int(c["b"])), max(int(c["a"]), int(c["b"]))) for c in self.connections)
        s = self.sensors
        cand = (s[lo] ^ s[hi]) & (body[lo] != body[hi]) & pair_passes(self.user_filters, self.filter_flags, connected, body, lo, hi)
        lo, hi = lo[cand], hi[cand]
        t = self.awake_tags
        touching = set(zip(np.minimum(t & np.uint64(0xffffffff), t >> np.uint64(32)).tolist(), np.maximum(t & np.uint64(0xffffffff), t >> np.uint64(32)).tolist()))
        tl, th = tag[lo], tag[hi]
        a = np.minimum(tl, th); b = np.maximum(tl, th)
        hit = np.array([(x, y) in touching for x, y in zip(a.tolist(), b.tolist())], bool) if len(a) else np.zeros(0, bool)
        out = np.zeros(int(hit.sum()), scenes.SENSOR_OVERLAP)
        out["tags"] = a[hit] | (b[hit] << np.uint64(32))
        lo_first = np.where(tl != th, tl < th, body[lo] < body[hi])   # equal tags: the lower body first
        first = np.where(lo_first, lo, hi)[hit]; second = np.where(lo_first, hi, lo)[hit]
        out["body_a"] = body[first]; out["body_b"] = body[second]
        return out[np.argsort(out["tags"], kind="stable")]

    def write_cached_impulses(self):
        super().write_cached_impulses()
        if self.sensors is not None:
            self._diff = (self.old, self.overlaps)
            self.old = self.overlaps.copy()

    def sensor_events(self, step):
        """The sensor events the last write_cached_impulses made, carrying `step`."""
        return overlap_events(self._diff[0], self._diff[1], step)


def add_sensors(s, zones=(), proximity=(), falling=(), proximity_radius=1.2):
    """A copy of scene `s` with sensor colliders: `zones` = (centre, half extents) static sensor boxes on body 0, appended after the boxes;
    `proximity` = bodies that get an extra sensor sphere of `proximity_radius` around their origin (the body's other colliders collide as
    before); `falling` = sphere indices of `s` made sensors (they overlap whatever they fall through).  Tags are renumbered: boxes
    0.., spheres after them, so every collider keeps a distinct tag."""
    t = s.copy()
    nz, npx = len(zones), len(proximity)
    g = scenes.Scene(s.n_bodies, s.n_boxes + nz, s.n_spheres + npx)
    for k in ("transforms", "properties", "momentum", "idle", "connections"):
        setattr(g, k, getattr(t, k))
    for k in ("time_step", "iterations", "gravity", "damping", "name", "filter_flags"):
        setattr(g, k, getattr(t, k))
    nb = s.n_boxes
    g.box_data[:nb] = t.box_data; g.box_transforms[:nb] = t.box_transforms
    for i, (c, h) in enumerate(zones):
        g.box_data["size"][nb + i] = h; g.box_transforms["position"][nb + i] = c; g.box_transforms["body"][nb + i] = 0
    ns = s.n_spheres
    g.sphere_data[:ns] = t.sphere_data; g.sphere_transforms[:ns] = t.sphere_transforms
    for i, b in enumerate(proximity):
        g.sphere_data["radius"][ns + i] = proximity_radius; g.sphere_transforms["body"][ns + i] = b
    g.box_tags[:] = np.arange(g.n_boxes, dtype=np.uint32)
    g.sphere_tags[:] = g.n_boxes + np.arange(g.n_spheres, dtype=np.uint32)
    sens = np.zeros(g.n_colliders, np.uint8)
    sens[nb:nb + nz] = 1
    sens[g.n_boxes + ns:] = 1
    sens[g.n_boxes + np.asarray(falling, np.int64)] = 1
    g.sensors = sens
    if t.collision_filters is not None:
        f = np.zeros(g.n_colliders, scenes.FILTER); f["category"] = 0xffff; f["mask"] = 0xffff
        f[:nb] = t.collision_filters[:nb]; f[g.n_boxes:g.n_boxes + ns] = t.collision_filters[nb:]
        g.collision_filters = f
    return g


def masked_out(s):
    """The same scene with every sensor collider given category 0 and mask 0 and no sensor table: the physics a sensor scene must have."""
    t = s.copy()
    f = t.collision_filters
    if f is None:
        f = np.zeros(t.n_colliders, scenes.FILTER); f["category"] = 0xffff; f["mask"] = 0xffff
    f = f.copy()
    on = np.asarray(t.sensors) != 0
    f["category"][on] = 0; f["mask"][on] = 0
    t.collision_filters, t.sensors = f, None
    return t
