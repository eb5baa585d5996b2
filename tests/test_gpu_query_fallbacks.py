"""Which scene queries fall back to testing every collider instead of walking the grid (nb_debug_read "ray_fallbacks", "overlap_fallbacks",
"shapecast_fallbacks"), query by query, against tests/golden/query_fallbacks.npz.  A change to a walk's margins, clip or cell caps can leave
every hit byte the same and still move these decisions, which decide what a query costs.  The recording: the query families of
tests/test_gpu_raycast.py, test_gpu_overlap.py and test_gpu_shapecast.py with their seeds, on the settled 8k-box pile, the mixed box /
sphere scene and the level-8 scene of sub-metre boxes and balls.  The families that may fall back (rays from far outside; overlap queries
far outside or larger than the scene; shape casts from far outside, larger than the scene or with rotations off unit length) are issued
one query per call, and each query's fallbacks are read from the counter's change (2 for an overlap query that falls back when
Sim.overlap repeats the call with room for all its hits); the other families are issued whole and their change is recorded.  A "ramp"
family per kind crosses the fallback thresholds on purpose: rays and sphere casts from 10^2 to 10^8 away, and overlap spheres from a tenth
of the scene to 30 times it, so the queries near a threshold pin the margins that decided them.  Each entry also holds a digest of the
queries it issued, so a changed scene shows as such.

    python tests/golden/make_query_fallbacks.py   (on an H100) records the golden file."""
import hashlib
import os
import numpy as np
import pytest
from nudge_b200 import abi, scenes
from tests.test_gpu_raycast import families as ray_families, small_mixed_scene, _settled
from tests.test_gpu_overlap import families as overlap_families
from tests.test_gpu_shapecast import families as cast_families

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "query_fallbacks.npz")
SCENES = (("pile8k", lambda: _settled(scenes.box_drop(8192, seed=4), 300), (11, 21, 31)),
          ("mixed", lambda: _settled(scenes.demo_scene(2000, 2000, iterations=8, spread=12.0, height=30.0, seed=6), 200), (12, 22, 32)),
          ("small_mixed", lambda: _settled(small_mixed_scene(), 150), (14, 23, 33)))
# kind: (family generator, the call, its counter, the families issued one query per call)
KINDS = {"ray": (ray_families, lambda sim, q: sim.raycast(q), "ray_fallbacks", ("far", "ramp")),
         "overlap": (overlap_families, lambda sim, q: sim.overlap(q), "overlap_fallbacks", ("large", "far", "ramp")),
         "shapecast": (cast_families, lambda sim, q: sim.shapecast(q), "shapecast_fallbacks", ("far", "large", "off_unit", "ramp"))}


def _ramp(kind, sim, rng, n=64):
    sim.download_bodies()
    p = sim.transforms["position"][1:]
    lo, hi = p.min(axis=0), p.max(axis=0)
    c, span = 0.5 * (lo + hi), float(np.linalg.norm(hi - lo))
    u = rng.normal(size=(n, 3)); u /= np.linalg.norm(u, axis=1, keepdims=True)
    if kind == "overlap":
        q = np.zeros(n, abi.OVERLAP_QUERY)
        q["shape"] = abi.OVERLAP_SPHERE; q["mask"] = 0xffffffff; q["ignore_body"] = abi.RAY_NO_HIT; q["rotation"][:, 3] = 1.0
        q["center"] = c + u; q["radius"] = span * 10.0 ** rng.uniform(-1.0, 1.5, n)
        return q
    dist = 10.0 ** rng.uniform(2.0, 8.0, n)[:, None]
    if kind == "ray":
        r = np.zeros(n, abi.RAY)
        r["mask"] = 0xffffffff; r["ignore_body"] = abi.RAY_NO_HIT; r["origin"] = c + u * dist; r["direction"] = -u; r["max_t"] = 2.0 * dist[:, 0]
        return r
    q = np.zeros(n, abi.SHAPE_CAST)
    q["shape"]["shape"] = abi.OVERLAP_SPHERE; q["shape"]["mask"] = 0xffffffff; q["shape"]["ignore_body"] = abi.RAY_NO_HIT
    q["shape"]["rotation"][:, 3] = 1.0; q["shape"]["radius"] = 0.5; q["shape"]["center"] = c + u * dist
    q["direction"] = -u; q["max_t"] = 2.0 * dist[:, 0]
    return q


def _digest(q):
    return np.frombuffer(hashlib.sha256(np.ascontiguousarray(q).tobytes()).digest()[:8], np.uint64)


def record():
    """{"scene/kind/family": per-query fallback bits or the family's count, "scene/kind/family/queries": the queries' digest}."""
    out = {}
    for scene, make, seeds in SCENES:
        sim = make()
        for (kind, (families, call, counter, single)), seed in zip(KINDS.items(), seeds):
            fam = families(sim, np.random.default_rng(seed))
            fam["ramp"] = _ramp(kind, sim, np.random.default_rng(seed + 100))
            for name, q in fam.items():
                key = "%s/%s/%s" % (scene, kind, name)
                calls = [q[k:k + 1] for k in range(len(q))] if name in single else [q]
                got = []
                for c in calls:
                    before = sim.debug_scalar(counter)
                    call(sim, c)
                    got.append(sim.debug_scalar(counter) - before)
                out[key] = np.array(got, np.uint32)
                out[key + "/queries"] = _digest(q)
        sim.close()
    return out


def test_fallback_decisions_equal_the_recording():
    want = dict(np.load(GOLDEN))
    got = record()
    assert sorted(got) == sorted(want)
    for key in sorted(k for k in got if not k.endswith("/queries")):
        assert got[key + "/queries"].tobytes() == want[key + "/queries"].tobytes(), key + ": the scene or the queries changed"
        bad = np.nonzero(got[key] != want[key])[0]
        assert not len(bad), (key, bad[:8], got[key][bad[:8]], want[key][bad[:8]])
