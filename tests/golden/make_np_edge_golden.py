"""Records tests/golden/np_edge_cases.npz: the unmodified reference (oracle/_ref/libnudge_ref.so, built by oracle/Makefile from the
reference's sources) run on the narrowphase edge-case scenes of tests/np_edge_cases.py.  Per scene it stores the full collide()
output in the reference's layout (count, contact data, bodies, 64-bit tags, sleeping pairs) and the stage digests of two full steps
(tests/parity_util.stage_digests), and prints a coverage table.  It fails if a case designed to touch makes no contact, if a case
designed to miss makes one, or if a family is missing from the table.

    python tests/golden/make_np_edge_golden.py"""
import os, sys
from collections import Counter, defaultdict
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import pyref  # noqa: E402
from tests import np_edge_cases as E  # noqa: E402
from tests.parity_util import stage_digests  # noqa: E402

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "np_edge_cases.npz")
STEPS = 2


def contact_cluster(es, tags):
    """Cluster of every contact, from the first collider tag in the reference's 64-bit tag (feature | a << 32 | b << 48)."""
    return es.cluster_of_tag()[((np.asarray(tags, np.uint64) >> np.uint64(32)) & np.uint64(0xffff)).astype(np.int64)]


def kind_of(c):
    return "-".join(sorted(col["shape"] for col in c["colliders"]))


def box_sphere_branch(c, data):
    """Which branch of box_sphere_collide (nudge.cpp:2523-2604) a contact came from, read off its normal in the box's frame."""
    if not len(data):
        return "none"
    b = c["colliders"][0] if c["colliders"][0]["shape"] == "box" else c["colliders"][1]
    qx, qy, qz, qw = np.asarray(b["rot"], np.float64)
    n = np.asarray(data[0]["normal"], np.float64)
    if not np.isfinite(n).all():
        return "corner/edge (non-finite normal)"
    local = E.qrot((-qx, -qy, -qz, qw), n) / max(np.linalg.norm((qx, qy, qz, qw)) ** 2, 1e-30)
    ax = np.nonzero(np.abs(local) > 1 - 1e-5)[0]
    return "face %s" % "xyz"[ax[0]] if len(ax) == 1 else "corner/edge"


def record(es):
    r = pyref.RefSim(es.scene, contact_capacity=max(1024, 16 * es.scene.n_colliders), arena_mb=256)
    r.collide()
    v = r.contacts_view()
    out = dict(count=np.array([v["count"]], np.uint32), data=v["data"], bodies_a=v["bodies"]["a"].astype(np.uint32),
               bodies_b=v["bodies"]["b"].astype(np.uint32), tags=v["tags"], sleeping=v["sleeping"], active=v["active"].astype(np.uint32),
               inputs=es.input_digest())
    r = pyref.RefSim(es.scene, contact_capacity=max(1024, 16 * es.scene.n_colliders), arena_mb=256)
    labels, d = stage_digests(r, False, STEPS, nan_blind=es.nan_blind)
    out["digests"] = d
    return out, labels


def main():
    arrays = {}
    pairs = Counter(); manifold = Counter(); branches = Counter(); families = defaultdict(Counter)
    n_sub = n_nan = 0
    bad = []
    for es in E.all_scenes():
        out, labels = record(es)
        for k, a in out.items():
            arrays["%s/%s" % (es.name, k)] = a
        data = out["data"]
        f = data.view(np.float32).reshape(len(data), -1) if len(data) else np.zeros((0, 8), np.float32)
        sub = (f != 0) & (np.abs(f) < np.finfo(np.float32).tiny)
        n_sub += int(sub.sum()); n_nan += int(np.isnan(f).sum())
        cl = contact_cluster(es, out["tags"])
        per = np.bincount(cl, minlength=len(es.clusters))
        for j, c in enumerate(es.clusters):
            k = kind_of(c)
            m = int(per[j])
            pairs[(k, "contact" if m else "no contact")] += 1
            if k == "box-box" and m:
                manifold[m] += 1
            if k == "box-sphere":
                branches[box_sphere_branch(c, data[cl == j])] += 1
            if es.name.startswith("tail"):
                continue
            families[c["family"]][m] += 1
            want = c["touch"]
            if (want is True and m == 0) or (want is False and m != 0) or (want not in (True, False) and m != want):
                bad.append("%s: %s case %d made %d contacts, designed for %s" % (es.name, c["family"], c["case"], m, want))
        print("%-10s %5d colliders %5d clusters %6d contacts" % (es.name, es.scene.n_colliders, len(es.clusters), len(data)), flush=True)
    print("\npairs per kind:")
    for (k, o), n in sorted(pairs.items()):
        print("  %-16s %-10s %6d" % (k, o, n))
    print("box-box contacts per manifold size:", " ".join("%d:%d" % (m, manifold[m]) for m in sorted(manifold)))
    print("box-sphere branch reached:", ", ".join("%s %d" % kv for kv in sorted(branches.items())))
    print("contact data values: %d subnormal, %d NaN" % (n_sub, n_nan))
    print("\nfamily (edge scenes): cases by contact count")
    for fam in sorted(families):
        print("  %-48s %s" % (fam, " ".join("%d:%d" % (m, n) for m, n in sorted(families[fam].items()))))
    missing = [m for m in range(1, 9) if not manifold[m]]
    if missing:
        bad.append("no box-box manifold of size %s" % missing)
    if bad:
        raise SystemExit("\n".join(bad))
    arrays["stage_labels"] = np.array(labels)
    np.savez_compressed(GOLDEN, **arrays)
    print("\nwrote", GOLDEN, os.path.getsize(GOLDEN), "bytes")


if __name__ == "__main__":
    main()
