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
With no table and no flag the result is the oracle's own, bit for bit (tests/test_collision_filter_oracle.py checks this over a run
with sleeping islands).  Contacts are matched to pairs by their collider tags, so scenes must give every collider a distinct tag."""
import numpy as np
from oracle import pyoracle


class Sets:
    """The oracle's union-find (oracle/nudge_oracle.cpp Sets): body 0, the static world, never joins."""

    def __init__(self, n):
        self.parent = list(range(n))

    def find(self, x):
        p = self.parent
        while p[x] != x:
            p[x] = p[p[x]]; x = p[x]
        return x

    def join(self, a, b):
        if not a or not b:
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
        s = self.scene
        idle = self.idle.copy()
        self.idle[:] = 0
        try:
            super().collide()
        finally:
            self.idle[:] = idle
        v = super().pairs_view()
        body = np.concatenate([self.box_transforms["body"], self.sphere_transforms["body"]]).astype(np.int64)
        tag = np.concatenate([self.box_tags, self.sphere_tags]).astype(np.uint64)
        lo, hi = v["lo"].astype(np.int64), v["hi"].astype(np.int64)
        conn = [(int(c["a"]), int(c["b"])) for c in self.connections]
        connected = set((min(a, b), max(a, b)) for a, b in conn)
        keep = pair_passes(self.filters, self.filter_flags, connected, body, lo, hi)
        lo, hi = lo[keep], hi[keep]
        self._pairs = dict(lo=v["lo"][keep].copy(), hi=v["hi"][keep].copy(), order=v["order"])
        B = s.n_bodies
        # coarse islands (nudge.cpp:3500-3703)
        sets = Sets(B)
        for a, b in conn:
            sets.join(a, b)
        ba, bb = body[lo], body[hi]
        for a, b in zip(ba.tolist(), bb.tolist()):
            sets.join(a, b)
        act = np.zeros(B, bool)
        for i in range(1, B):
            if idle[i] != 0xff:
                act[sets.find(i)] = True
        sleeping, live = [], set()
        for a, b, x, y in zip(ba.tolist(), bb.tolist(), lo.tolist(), hi.tolist()):
            if a == b:
                continue
            if act[sets.find(a) if a else sets.find(b)]:
                live.add((min(int(tag[x]), int(tag[y])), max(int(tag[x]), int(tag[y]))))
            else:
                ta, tb = int(tag[x]), int(tag[y])
                sleeping.append(ta | (tb << 32) if ta > tb else tb | (ta << 32))
        # the live pairs' contacts, in the oracle's order
        n = self.contacts.count
        tags = self.contact_tags[:n]
        t0, t1 = (tags & np.uint64(0xffffffff)).astype(np.int64), (tags >> np.uint64(32)).astype(np.int64)
        sel = np.array([(min(a, b), max(a, b)) in live for a, b in zip(t0.tolist(), t1.tolist())], bool) if n else np.zeros(0, bool)
        data, bodies, tags, feats = self.contact_data[:n][sel], self.contact_bodies[:n][sel], tags[sel], self.contact_features[:n][sel]
        # fine islands, active bodies, contact compaction (nudge.cpp:3788-4006)
        sets = Sets(B)
        for a, b in conn:
            sets.join(a, b)
        for a, b in zip(bodies["a"].tolist(), bodies["b"].tolist()):
            sets.join(a, b)
        act = np.zeros(B, bool)
        for i in range(1, B):
            if idle[i] != 0xff:
                act[sets.find(i)] = True
        active = [i for i in range(1, B) if act[sets.find(i)]]
        out = np.zeros(len(tags), bool)
        i = 0
        while i < len(tags):
            j = i
            while j < len(tags) and tags[j] == tags[i]:
                j += 1
            a, b = int(bodies["a"][i]), int(bodies["b"][i])
            if act[sets.find(a) if a else sets.find(b)]:
                out[i:j] = True
            else:
                sleeping.append(int(tags[i]))
            i = j
        m = int(out.sum())
        self.contact_data[:m] = data[out]; self.contact_bodies[:m] = bodies[out]; self.contact_tags[:m] = tags[out]; self.contact_features[:m] = feats[out]
        self.contacts.count = m
        sl = np.sort(np.array(sleeping, np.uint64))
        self.sleeping_pairs[:len(sl)] = sl
        self.contacts.sleeping_count = len(sl)
        self.active_indices[:len(active)] = active
        self.active.count = len(active)

    def pairs_view(self):
        return dict(self._pairs)
