"""Test infrastructure (no device): collider tags as applications assign them, and custom contacts appended after collide.

The scene generators number their tags 0..K-1, so the largest tag is always about the collider count.  The step's contact key layout
depends on the tag width, which nb_upload_colliders derives from the largest tag, so these helpers retag a scene:

  - monotone(scene, bits):  a strictly increasing map f of the dense tags whose largest value has exactly `bits` bits.  No tag comparison
    changes, so the run must equal the dense twin's bit for bit, every tag mapped through f (TagMap).
  - permuted(scene, seed):  a random injective assignment; the ground no longer carries the smallest tag.
  - shared(scene, merge):   duplicate tags: all colliders of a body share one tag, and the given collider pairs share one too.

layout(tagbits, internal) restates read_sort's key layout (nudge_b200/csrc/nb_api.cu) so that each case can assert the layout it reaches."""
import numpy as np
from nudge_b200 import scenes

MASK32 = np.uint64(0xffffffff)
S32 = np.uint64(32)


def bits_for(n):
    """nb_api.cu bits_for: the least b >= 1 with 2^b >= n."""
    b = 1
    while (1 << b) < n:
        b += 1
    return b


def collider_tags(scene):
    return np.concatenate([scene.box_tags, scene.sphere_tags]).astype(np.uint64)


def tagbits(scene):
    """The width nb_upload_colliders derives: bits_for(max(1, largest tag) + 1)."""
    t = collider_tags(scene)
    return bits_for(max(1, int(t.max()) if len(t) else 1) + 1)


def layout(tb, internal=True):
    """read_sort's key layout for `tb` tag bits: 'packed' (B | A | 16 feature bits, one sort), 'spread' (the same with keys of B < 8
    stretched over one more bit) or 'two-pass' (a 32-bit sort on the feature word, then a sort over the pair word).  Contacts uploaded
    with nb_upload_contacts (internal=False) always take the two-pass path."""
    if internal and 2 * tb + 16 <= 64:
        return "spread" if tb >= 3 and 2 * tb + 17 <= 64 else "packed"
    return "two-pass"


def key_bits(tb, internal=True):
    """Bits the contact-order sort(s) of that layout cover."""
    lay = layout(tb, internal)
    return {"packed": (2 * tb + 16,), "spread": (2 * tb + 17,), "two-pass": (32, 2 * tb)}[lay]


class TagMap:
    """f as a table over the dense tags, applied to collider tags and, half by half, to 64-bit pair keys A | B << 32 (contact, cache,
    sleeping-pair, sensor-overlap and event tags)."""

    def __init__(self, f):
        self.f = np.asarray(f, np.uint64)

    def tag(self, t):
        return self.f[np.asarray(t, np.int64)]

    def pair(self, t):
        t = np.asarray(t, np.uint64)
        return self.f[(t & MASK32).astype(np.int64)] | (self.f[(t >> S32).astype(np.int64)] << S32)

    def apply(self, scene):
        """A copy of `scene` with every collider tag mapped."""
        s = scene.copy()
        s.box_tags[:] = self.tag(scene.box_tags).astype(np.uint32)
        s.sphere_tags[:] = self.tag(scene.sphere_tags).astype(np.uint32)
        return s


def _dense(scene):
    t = collider_tags(scene)
    assert np.array_equal(np.sort(t), np.arange(len(t))), "retagging starts from the generators' dense tags 0..K-1"
    return len(t)


def monotone(scene, bits, seed=0):
    """(retagged scene, TagMap): f strictly increasing on 0..K-1, f(0) < 8 (so the packed layout's stretch of B < 8 has work), and
    f(K-1) = 2^bits - 1, so that the width nb_upload_colliders derives is exactly `bits`."""
    k = _dense(scene)
    top = (1 << bits) - 1
    assert k <= top + 1, "%d colliders do not fit %d tag bits" % (k, bits)
    rng = np.random.default_rng(seed)
    if k == 1:
        f = np.array([top], np.uint64)
    else:
        lo = int(rng.integers(0, min(8, top - k + 2)))
        mid = np.sort(rng.choice(top - lo - 1, k - 2, replace=False).astype(np.uint64)) + np.uint64(lo + 1) if k > 2 else np.zeros(0, np.uint64)
        f = np.concatenate([[np.uint64(lo)], mid, [np.uint64(top)]]).astype(np.uint64)
    assert (np.diff(f.astype(np.float64)) > 0).all() and int(f[-1]) == top
    m = TagMap(f)
    return m.apply(scene), m


def permuted(scene, seed, max_tag=0xffff):
    """(retagged scene, TagMap): distinct tags drawn at random from 0..max_tag, max_tag itself included, the ground's not the smallest."""
    k = _dense(scene)
    rng = np.random.default_rng(seed)
    f = rng.choice(max_tag, k - 1, replace=False).astype(np.uint64)
    f = np.concatenate([f, [np.uint64(max_tag)]])
    f = f[rng.permutation(k)]
    if k > 1 and f[0] == f.min():
        j = int(rng.integers(1, k))
        f[0], f[j] = f[j], f[0]
    m = TagMap(f)
    return m.apply(scene), m


def compound(scene, bodies, radius_scale=0.45):
    """A copy of `scene` with one extra sphere collider on each of `bodies` (a box body): a body of two colliders.  The sphere sits at the
    box's centre inside it, so it only adds contacts where the box already touches; tags stay dense (spheres after boxes)."""
    bodies = np.asarray(bodies, np.int64)
    box_of = {int(b): i for i, b in enumerate(scene.box_transforms["body"])}
    g = scenes.Scene(scene.n_bodies, scene.n_boxes, scene.n_spheres + len(bodies))
    for k, v in scene.__dict__.items():
        if k not in ("sphere_tags", "sphere_data", "sphere_transforms"):
            setattr(g, k, v.copy() if isinstance(v, np.ndarray) else v)
    ns = scene.n_spheres
    g.sphere_data[:ns] = scene.sphere_data; g.sphere_transforms[:ns] = scene.sphere_transforms
    for i, b in enumerate(bodies):
        g.sphere_data["radius"][ns + i] = radius_scale * float(scene.box_data["size"][box_of[int(b)]].min())
        g.sphere_transforms["body"][ns + i] = b
    g.box_tags[:] = np.arange(g.n_boxes, dtype=np.uint32)
    g.sphere_tags[:] = g.n_boxes + np.arange(g.n_spheres, dtype=np.uint32)
    g.name = scene.name + "_compound"
    return g


def shared(scene, group=2):
    """A copy of `scene` with duplicate tags: every collider carries the tag (body + group - 1) // group, so all colliders of a body share
    one, the static world keeps 0 alone, and `group` neighbouring bodies (unrelated otherwise) share one."""
    s = scene.copy()
    body = np.concatenate([s.box_transforms["body"], s.sphere_transforms["body"]]).astype(np.uint32)
    tag = (body + np.uint32(group - 1)) // np.uint32(group)
    s.box_tags[:] = tag[:s.n_boxes]; s.sphere_tags[:] = tag[s.n_boxes:]
    s.name = scene.name + "_shared"
    return s


def equal_tag_contacts(tags):
    """How many contacts (widened tags A | B << 32) have A == B."""
    t = np.asarray(tags, np.uint64)
    return int(((t & MASK32) == (t >> S32)).sum())


# ---- custom contacts appended after collide (example/main.cpp:288: "custom contacts can be added here") ----
CUSTOM = np.dtype([("data", scenes.CONTACT), ("a", "<u4"), ("b", "<u4"), ("A", "<u4"), ("B", "<u4"), ("feature", "<u4")])


def custom_contacts(sim, step, high_tags, seed=0, n_ground=4, n_pair=3):
    """Custom contacts for the sim's current state (a pure function of its host arrays, so the same on every implementation that holds the
    same state): `n_ground` awake bodies resting on body 0 and `n_pair` pairs of awake bodies, with tags from `high_tags` (values no
    collider need carry) and arbitrary feature words.  Both tag orders occur (A > B and A < B)."""
    rng = np.random.default_rng(seed * 1000 + step)
    act = np.asarray(sim.active_indices[:sim.active.count], np.int64)
    act = act[act != 0]
    if len(act) < 2:
        return np.zeros(0, CUSTOM)
    pick = rng.choice(act, min(len(act), n_ground + 2 * n_pair), replace=False)
    rows = np.zeros(len(pick), CUSTOM)
    hi = np.asarray(high_tags, np.uint64)
    k = 0
    for b in pick[:n_ground]:
        rows[k]["a"], rows[k]["b"] = b, 0
        k += 1
    rest = pick[n_ground:]
    for i in range(len(rest) // 2):
        rows[k]["a"], rows[k]["b"] = rest[2 * i], rest[2 * i + 1]
        k += 1
    rows = rows[:k]
    pos = sim.transforms["position"][rows["a"].astype(np.int64)]
    rows["data"]["position"] = pos - np.float32(0.25) * np.array([0, 1, 0], np.float32)
    rows["data"]["penetration"] = np.float32(0.004)
    rows["data"]["normal"] = np.array([0, 1, 0], np.float32)
    rows["data"]["friction"] = np.float32(0.5)
    rows["A"] = hi[rng.integers(0, len(hi), k)]
    rows["B"] = hi[rng.integers(0, len(hi), k)] - rng.integers(0, 3, k).astype(np.uint64)
    rows["feature"] = rng.integers(0, 1 << 32, k, dtype=np.uint64).astype(np.uint32)
    return rows


def append_wide(sim, rows):
    """Appends `rows` to a widened-layout host contact set (OracleSim, Sim after download_contacts)."""
    n, k = sim.contacts.count, len(rows)
    assert n + k <= sim.cap
    sim.contact_data[n:n + k] = rows["data"]
    sim.contact_bodies["a"][n:n + k] = rows["a"]; sim.contact_bodies["b"][n:n + k] = rows["b"]
    sim.contact_tags[n:n + k] = rows["A"].astype(np.uint64) | (rows["B"].astype(np.uint64) << S32)
    sim.contact_features[n:n + k] = rows["feature"]
    sim.contacts.count = n + k


def append_ref(sim, rows):
    """Appends `rows` to the reference's uint16-layout host contact set (pyref.RefSim): tag = feature | A << 32 | B << 48."""
    assert (rows["A"] <= 0xffff).all() and (rows["B"] <= 0xffff).all()
    n, k = sim.contacts.count, len(rows)
    assert n + k <= sim.cap
    sim.contact_data[n:n + k] = rows["data"]
    sim.contact_bodies["a"][n:n + k] = rows["a"]; sim.contact_bodies["b"][n:n + k] = rows["b"]
    sim.contact_tags[n:n + k] = rows["feature"].astype(np.uint64) | (rows["A"].astype(np.uint64) << S32) | (rows["B"].astype(np.uint64) << np.uint64(48))
    sim.contacts.count = n + k
