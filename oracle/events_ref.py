"""TEST INFRASTRUCTURE ONLY: numpy restatement of the contact-event contract (nb_contact_event, include/nudge_b200.h; DESIGN.md §8.5).

Written from the contract, not from the kernels: a pair (key A | B << 32) is touching after a step if the cache that step wrote holds
an entry with that key.  With `old` = the cache before write_cached_impulses, `cur` = the step's contacts and `culled` = the kept
entries of sleeping pairs: END = in old, not in cur, not in culled; BEGIN = in cur, not in old.  ENDs come first, then BEGINs, each in
ascending key order.  Only tests may import this."""
import numpy as np
from nudge_b200 import scenes as S


def events(old_tags, contacts, impulses, culled_tags, step):
    """The events of one write_cached_impulses.  contacts: a contacts_view() dict (tags, features, data, bodies) in any order;
    impulses: (n, 3) float32, the final cached impulse of each of those contacts; step: the value the events carry."""
    tags = np.asarray(contacts["tags"], np.uint64)
    features = np.asarray(contacts["features"], np.uint32)
    order = np.lexsort((features, tags))   # (tag, feature) order
    pairs = {}
    for c in order:
        pairs.setdefault(int(tags[c]), []).append(int(c))
    old = set(int(t) for t in np.asarray(old_tags, np.uint64))
    culled = set(int(t) for t in np.asarray(culled_tags, np.uint64))
    ends = sorted(old - set(pairs) - culled)
    begins = sorted(set(pairs) - old)
    out = np.zeros(len(ends) + len(begins), S.CONTACT_EVENT)
    out["step"] = step
    for k, t in enumerate(ends):
        out[k]["tags"] = t
        out[k]["kind"] = S.CONTACT_END
    data, bodies = contacts["data"], contacts["bodies"]
    imp = np.asarray(impulses, np.float32)
    for k, t in enumerate(begins, len(ends)):
        cs = pairs[t]
        deepest = cs[0]
        acc = [np.float32(0.0)] * 3
        for c in cs:
            if data[c]["penetration"] > data[deepest]["penetration"]:   # strictly deeper; False for a NaN on either side
                deepest = c
            acc = [np.float32(acc[i] + imp[c, i]) for i in range(3)]   # sequential fp32 sum in (tag, feature) order
        e = out[k]
        e["tags"] = t; e["kind"] = S.CONTACT_BEGIN
        e["body_a"] = bodies[deepest]["a"]; e["body_b"] = bodies[deepest]["b"]; e["contacts"] = len(cs)
        e["penetration"] = data[deepest]["penetration"]; e["position"] = data[deepest]["position"]; e["normal"] = data[deepest]["normal"]
        e["impulse"] = acc
    return out


def cache_impulses(tags, features, cache):
    """Impulse of every contact (tags[i], features[i]) = the entry with the same (tag, feature) in `cache` (a cache_view() dict)."""
    at = {(int(t), int(f)): i for i, (t, f) in enumerate(zip(cache["tags"], cache["features"]))}
    idx = np.array([at[(int(t), int(f))] for t, f in zip(tags, features)], np.int64)
    return cache["data"]["impulse"][idx] if len(idx) else np.zeros((0, 3), np.float32)


def touching(cache):
    """The distinct pair keys of a cache_view() dict."""
    return set(int(t) for t in cache["tags"])


class OracleEvents:
    """Steps an OracleSim stage by stage and returns the events of each step, with the device's step counter (0 at enable)."""

    def __init__(self, oracle):
        self.o = oracle
        self.step_index = 0

    def step(self):
        o = self.o
        o.collide(); o.apply_gravity_damping(); o.read_cached_impulses(); o.setup_contact_constraints()
        for _ in range(int(o.scene.iterations)):
            o.apply_impulses()
        o.update_cached_impulses()
        old = o.cache_view()
        cur = o.contacts_view()
        culled = o.impulses_view()["culled_tags"]
        o.write_cached_impulses()
        new = o.cache_view()
        o.advance()
        ev = events(old["tags"], cur, cache_impulses(cur["tags"], cur["features"], new), culled, self.step_index)
        self.step_index += 1
        return ev
