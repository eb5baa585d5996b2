"""Records tests/golden/broadphase_edges.npz: the unmodified reference (oracle/_ref/libnudge_ref.so, built by oracle/Makefile from the
reference's sources) run for two full steps on every broadphase edge-case scene of tests/broadphase_edges.py that fits it, as stage
digests (tests/parity_util.stage_digests), with a digest of each scene's inputs so that a changed scene is caught.

    python tests/golden/make_broadphase_golden.py"""
import os, sys
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import pyref  # noqa: E402
from tests import broadphase_edges as E, grid_ref  # noqa: E402
from tests.parity_util import stage_digests  # noqa: E402

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "broadphase_edges.npz")
STEPS = 2


def main():
    out = {}
    for es in E.all_scenes(grid_ref.host_rcp()):
        if not es.scene.fits_reference() or es.kind not in ("plain", "dynamic"):
            continue
        labels, d = stage_digests(pyref.RefSim(es.scene, contact_capacity=E.CAPACITY, arena_mb=512), False, STEPS)
        out[es.name + "/digests"] = d
        out[es.name + "/inputs"] = E.input_digest(es.scene)
        out["stage_labels"] = np.array(labels)
        print("%-24s %d stages" % (es.name, len(d)))
    np.savez_compressed(GOLDEN, **out)


if __name__ == "__main__":
    main()
