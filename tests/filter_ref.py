"""Test infrastructure: the collide stage with collision filters (include/nudge_b200.h nb_upload_collision_filters), restated on top of the
unmodified widened CPU oracle.

The filter only takes pairs out of the broadphase list, and everything else in nbo_collide is a function of that list:
  - the oracle is run with every body awake, which gives the full sorted pair list and every pair's contacts in pipeline order (box-box
    face contacts, box-box edge contacts, box-sphere, sphere-sphere, each in pair order) with nothing removed by the island passes;
  - the rejected pairs are taken out of that list, and the two island passes of nudge.cpp:3500-3703 / 3788-3971 are restated here on the
    real idle counters: coarse islands over connections and the kept pairs give the sleeping pairs and the live pairs, the live pairs' contacts
    keep their order, fine islands over connections and those contacts give the active bodies and the contacts of sleeping fine islands
    (appended to the sleeping pairs, one tag per pair), and the sleeping pairs are sorted (nudge.cpp:4008).
A pair's contacts depend only on its two colliders, so dropping pairs leaves the others' contacts and their relative order unchanged.
restate_collide does this for any pair rule, and with the kinematic island rules for tests/kinematic_ref.py.
With no table and no flag the result is the oracle's own, bit for bit (tests/test_collision_filter_oracle.py checks this over a run
with sleeping islands).  Contacts are matched to pairs by their collider tags, so scenes must give every collider a distinct tag."""
import numpy as np
from oracle import pyoracle


class Sets:
    """The oracle's union-find (oracle/nudge_oracle.cpp Sets): body 0, the static world, never joins, and neither do the bodies in
    `fixed` (kinematic bodies, tests/kinematic_ref.py)."""

    def __init__(self, n, fixed=()):
        self.parent = list(range(n))
        self.fixed = fixed

    def find(self, x):
        p = self.parent
        while p[x] != x:
            p[x] = p[p[x]]; x = p[x]
        return x

    def join(self, a, b):
        if not a or not b or a in self.fixed or b in self.fixed:
            return
        a, b = self.find(a), self.find(b)
        if a != b:
            self.parent[max(a, b)] = min(a, b)


def pair_passes(filters, flags, connected, body, lo, hi):
    """Per pair (collider indices lo, hi): the category / mask rule and, with flag 1, the connected opt-out."""
    keep = np.ones(len(lo), bool)
    if filters is not None:
        cat, mask = filters["category"], filters["mask"]
        keep &= ((cat[lo] & mask[hi]) != 0) & ((cat[hi] & mask[lo]) != 0)
    if flags & 1 and connected:
        keep &= np.array([(min(a, b), max(a, b)) not in connected for a, b in zip(body[lo].tolist(), body[hi].tolist())], bool)
    return keep


def restate_collide(sim, run_oracle, pair_keep, kin=(), moving=()):
    """The collide stage of `sim` restated from the all-awake oracle run `run_oracle()` (module docstring).  `pair_keep(body, lo, hi)` is the
    mask of the broadphase pairs kept (collider indices lo, hi; body = each collider's body).  `kin` are the kinematic bodies, which never
    join a set, and `moving` those of them that move: each is active itself and makes the dynamic side of each of its edges active.  With
    `kin` empty these are the oracle's island rules.  Records the all-awake run's pair list and contact tags as sim.awake_pairs and
    sim.awake_tags, and the kept pairs for pairs_view as sim._pairs."""
    idle = sim.idle.copy()
    sim.idle[:] = 0
    try:
        run_oracle()
    finally:
        sim.idle[:] = idle
    v = pyoracle.OracleSim.pairs_view(sim)
    sim.awake_pairs = v
    sim.awake_tags = sim.contact_tags[:sim.contacts.count].copy()
    body = np.concatenate([sim.box_transforms["body"], sim.sphere_transforms["body"]]).astype(np.int64)
    tag = np.concatenate([sim.box_tags, sim.sphere_tags]).astype(np.uint64)
    lo, hi = v["lo"].astype(np.int64), v["hi"].astype(np.int64)
    keep = pair_keep(body, lo, hi)
    lo, hi = lo[keep], hi[keep]
    sim._pairs = dict(lo=v["lo"][keep].copy(), hi=v["hi"][keep].copy(), order=v["order"])
    B = sim.scene.n_bodies
    nondyn = set(kin) | {0}
    conn = [(int(c["a"]), int(c["b"])) for c in sim.connections]

    def islands(edges):
        sets = Sets(B, kin)
        for a, b in edges:
            sets.join(a, b)
        act = np.zeros(B, bool)
        for i in range(1, B):
            if i in kin:
                act[i] = i in moving
            elif idle[i] != 0xff:
                act[sets.find(i)] = True
        for a, b in edges:   # the taint of a moving kinematic body
            if a in moving and b not in nondyn:
                act[sets.find(b)] = True
            elif b in moving and a not in nondyn:
                act[sets.find(a)] = True
        return sets, act

    def set_of(sets, a, b):
        return sets.find(a) if a not in nondyn else sets.find(b)

    # coarse islands (nudge.cpp:3500-3703)
    ba, bb = body[lo], body[hi]
    sets, act = islands(conn + list(zip(ba.tolist(), bb.tolist())))
    sleeping, live = [], set()
    for a, b, x, y in zip(ba.tolist(), bb.tolist(), lo.tolist(), hi.tolist()):
        if a == b:
            continue
        if act[set_of(sets, a, b)]:
            live.add((min(int(tag[x]), int(tag[y])), max(int(tag[x]), int(tag[y]))))
        else:
            ta, tb = int(tag[x]), int(tag[y])
            sleeping.append(ta | (tb << 32) if ta > tb else tb | (ta << 32))
    # the live pairs' contacts, in the oracle's order
    n = sim.contacts.count
    tags = sim.contact_tags[:n]
    t0, t1 = (tags & np.uint64(0xffffffff)).astype(np.int64), (tags >> np.uint64(32)).astype(np.int64)
    sel = np.array([(min(a, b), max(a, b)) in live for a, b in zip(t0.tolist(), t1.tolist())], bool) if n else np.zeros(0, bool)
    data, bodies, tags, feats = sim.contact_data[:n][sel], sim.contact_bodies[:n][sel], tags[sel], sim.contact_features[:n][sel]
    # fine islands, active bodies, contact compaction (nudge.cpp:3788-4006)
    sets, act = islands(conn + list(zip(bodies["a"].tolist(), bodies["b"].tolist())))
    active = [i for i in range(1, B) if (act[i] if i in kin else act[sets.find(i)])]
    out = np.zeros(len(tags), bool)
    i = 0
    while i < len(tags):
        j = i
        while j < len(tags) and tags[j] == tags[i]:
            j += 1
        a, b = int(bodies["a"][i]), int(bodies["b"][i])
        if act[set_of(sets, a, b)]:
            out[i:j] = True
        else:
            sleeping.append(int(tags[i]))
        i = j
    m = int(out.sum())
    sim.contact_data[:m] = data[out]; sim.contact_bodies[:m] = bodies[out]; sim.contact_tags[:m] = tags[out]; sim.contact_features[:m] = feats[out]
    sim.contacts.count = m
    sl = np.sort(np.array(sleeping, np.uint64))
    sim.sleeping_pairs[:len(sl)] = sl
    sim.contacts.sleeping_count = len(sl)
    sim.active_indices[:len(active)] = active
    sim.active.count = len(active)


class FilteredOracleSim(pyoracle.OracleSim):
    """OracleSim whose collide stage applies the scene's (or the uploaded) collision filters; every later stage is the oracle's own."""

    def __init__(self, scene, ftz=False, contact_capacity=None):
        super().__init__(scene, ftz, contact_capacity)
        self.upload_collision_filters(getattr(scene, "collision_filters", None), getattr(scene, "filter_flags", 0))

    def upload_collision_filters(self, filters, flags=0):
        """Mirror of Sim.upload_collision_filters: None (or empty) removes the table; flags & 1 = FILTER_SKIP_CONNECTED."""
        self.filters = None if filters is None or len(filters) == 0 else np.array(filters, copy=True)
        self.filter_flags = int(flags)

    def collide(self):
        connected = set((min(int(c["a"]), int(c["b"])), max(int(c["a"]), int(c["b"]))) for c in self.connections)
        restate_collide(self, super().collide, lambda body, lo, hi: pair_passes(self.filters, self.filter_flags, connected, body, lo, hi))

    def pairs_view(self):
        return dict(self._pairs)
