"""Restatement of nb_remove_bodies / nb_add_bodies (include/nudge_b200.h, DESIGN.md section 8.10) on host arrays, in numpy.

remove_bodies(scene, idx, cache, rows, old_overlaps) applies the header's rule to a scenes.Scene whose transforms, momentum and idle counters
hold the current state: the wake set (contact-cache keys that pair a kept collider's tag with a removed collider's tag, and connections to a
removed body; never body 0 or a kinematic body), then the stable compaction of bodies, colliders, connections, the filter / sensor tables,
the kinematic set, the user rows and the sensor overlap list.  add_bodies(scene, fragment) appends a fragment (its collider bodies count from
its own first body, its collision_filters / sensors rows are the added colliders' table entries)."""
import numpy as np
from nudge_b200 import scenes

REMOVED = np.uint32(0xffffffff)


def body_map(n_bodies, idx):
    """Old index -> new index, REMOVED for the removed bodies."""
    keep = np.ones(n_bodies, bool)
    keep[np.asarray(idx, np.int64)] = False
    m = np.full(n_bodies, REMOVED, np.uint32)
    m[keep] = np.arange(int(keep.sum()), dtype=np.uint32)
    return keep, m


def wake_set(scene, keep, cache_tags):
    """Bodies woken by the removal (a bool mask over the old bodies)."""
    bodies = np.concatenate([scene.box_transforms["body"], scene.sphere_transforms["body"]]).astype(np.int64)
    tags = np.concatenate([scene.box_tags, scene.sphere_tags]).astype(np.int64)
    wake = np.zeros(scene.n_bodies, bool)
    removed_tags = set(tags[~keep[bodies]].tolist())
    by_tag = {}
    for t, b in zip(tags.tolist(), bodies.tolist()):
        if keep[b]:
            by_tag.setdefault(t, []).append(b)
    for key in np.asarray(cache_tags if cache_tags is not None else [], np.uint64).tolist():
        a, b = key & 0xffffffff, key >> 32
        if b in removed_tags:
            wake[by_tag.get(a, [])] = True
        if a in removed_tags:
            wake[by_tag.get(b, [])] = True
    for a, b in zip(scene.connections["a"].tolist(), scene.connections["b"].tolist()):
        if not keep[a] and keep[b]:
            wake[b] = True
        if not keep[b] and keep[a]:
            wake[a] = True
    wake[0] = False
    if scene.kinematic is not None:
        wake[scene.kinematic["body"].astype(np.int64)] = False
    return wake


def remove_bodies(scene, idx, cache=None, rows=None, old_overlaps=None):
    """Returns (new scene, new rows, new overlap list, woken mask over the old bodies).  `cache` = the cache's keys (u64 tags)."""
    s = scene
    keep, m = body_map(s.n_bodies, idx)
    woken = wake_set(s, keep, cache)
    out = s.copy()
    idle = s.idle.copy()
    idle[woken] = 0
    out.transforms, out.properties, out.momentum, out.idle = s.transforms[keep].copy(), s.properties[keep].copy(), s.momentum[keep].copy(), idle[keep]
    kb = keep[s.box_transforms["body"].astype(np.int64)]
    ks = keep[s.sphere_transforms["body"].astype(np.int64)]
    out.box_tags, out.box_data, out.box_transforms = s.box_tags[kb].copy(), s.box_data[kb].copy(), s.box_transforms[kb].copy()
    out.sphere_tags, out.sphere_data, out.sphere_transforms = s.sphere_tags[ks].copy(), s.sphere_data[ks].copy(), s.sphere_transforms[ks].copy()
    out.box_transforms["body"] = m[out.box_transforms["body"].astype(np.int64)]
    out.sphere_transforms["body"] = m[out.sphere_transforms["body"].astype(np.int64)]
    kc = np.concatenate([kb, ks])
    if s.collision_filters is not None:
        out.collision_filters = s.collision_filters[kc].copy()
    if s.sensors is not None:
        out.sensors = s.sensors[kc].copy()
    c = s.connections
    kconn = keep[c["a"].astype(np.int64)] & keep[c["b"].astype(np.int64)]
    out.connections = c[kconn].copy()
    out.connections["a"] = m[out.connections["a"].astype(np.int64)]
    out.connections["b"] = m[out.connections["b"].astype(np.int64)]
    if s.kinematic is not None:
        k = s.kinematic[keep[s.kinematic["body"].astype(np.int64)]].copy()
        k["body"] = m[k["body"].astype(np.int64)]
        out.kinematic = k if len(k) else None
    new_rows = None
    if rows is not None:
        r = rows[keep[rows["a"].astype(np.int64)] & keep[rows["b"].astype(np.int64)]].copy()
        r["a"] = m[r["a"].astype(np.int64)]; r["b"] = m[r["b"].astype(np.int64)]
        new_rows = r
    new_ov = None
    if old_overlaps is not None:
        new_ov = old_overlaps.copy()
        for f in ("body_a", "body_b"):
            v = new_ov[f]
            ok = v != REMOVED
            v[ok] = m[v[ok].astype(np.int64)]
    return out, new_rows, new_ov, woken


def add_bodies(scene, fragment):
    """The scene with `fragment` appended (a new scene)."""
    s, fr = scene, fragment
    B = s.n_bodies
    out = s.copy()
    for k in ("transforms", "properties", "momentum", "idle"):
        setattr(out, k, np.concatenate([getattr(s, k), getattr(fr, k)]))
    bx, sx = fr.box_transforms.copy(), fr.sphere_transforms.copy()
    bx["body"] += np.uint32(B); sx["body"] += np.uint32(B)
    out.box_tags, out.box_data, out.box_transforms = np.concatenate([s.box_tags, fr.box_tags]), np.concatenate([s.box_data, fr.box_data]), np.concatenate([s.box_transforms, bx])
    out.sphere_tags, out.sphere_data = np.concatenate([s.sphere_tags, fr.sphere_tags]), np.concatenate([s.sphere_data, fr.sphere_data])
    out.sphere_transforms = np.concatenate([s.sphere_transforms, sx])
    nb, fb = s.n_boxes, fr.n_boxes
    if s.collision_filters is not None:
        f = fr.collision_filters
        out.collision_filters = np.concatenate([s.collision_filters[:nb], f[:fb], s.collision_filters[nb:], f[fb:]])
    if s.sensors is not None:
        f = fr.sensors
        out.sensors = np.concatenate([s.sensors[:nb], f[:fb], s.sensors[nb:], f[fb:]])
    return out


def rebuild_oracle(o, scene):
    """A new OracleSim on `scene` that keeps `o`'s contact cache (the cache is not part of the edit)."""
    from oracle import pyoracle
    o2 = pyoracle.OracleSim(scene, contact_capacity=o.cap)
    n = o.cache.count
    o2.cache_tags[:n] = o.cache_tags[:n]; o2.cache_features[:n] = o.cache_features[:n]; o2.cache_data[:n] = o.cache_data[:n]
    o2.cache.count = n
    return o2


def live_scene(x):
    """x.scene with x's current transforms, momentum and idle counters (x: a Sim after download_bodies, or an OracleSim)."""
    s = x.scene.copy()
    s.transforms, s.momentum, s.idle = x.transforms.copy(), x.momentum.copy(), x.idle.copy()
    s.properties = x.properties.copy()
    return s
