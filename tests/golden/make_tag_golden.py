"""Records tests/golden/tag_cases.npz: the unmodified reference (oracle/_ref/libnudge_ref.so, built by oracle/Makefile from the reference's
sources) run through the scenarios of tests/test_tags_ref.py (permuted, sparse and shared collider tags, custom contacts), one 8-byte
SHA-256 digest per stage.

    python tests/golden/make_tag_golden.py"""
import os, sys
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import pyref  # noqa: E402
from tests import test_tags_ref as T  # noqa: E402


def main():
    out = {}
    for name, case in sorted(T.CASES.items()):
        out[name] = case(lambda scene, cap: pyref.RefSim(scene, contact_capacity=cap, arena_mb=1024), False)[1]
        print(name, len(out[name]), "stage digests", flush=True)
    np.savez_compressed(T.GOLDEN, **out)
    print("wrote", T.GOLDEN)


if __name__ == "__main__":
    main()
