"""Records tests/golden/query_fallbacks.npz: which scene queries of tests/test_gpu_query_fallbacks.py fall back to testing every collider,
query by query (see that module).  Needs an H100 and the built library.  The committed file was recorded with the library of commit
723db74, before the scene queries shared their walk, so the test holds the shared walk to the decisions of the three walks it replaced.

    python tests/golden/make_query_fallbacks.py"""
import os, sys
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from tests import test_gpu_query_fallbacks as T  # noqa: E402


def main():
    out = T.record()
    for key in sorted(k for k in out if not k.endswith("/queries")):
        print(key, len(out[key]), "calls", int(out[key].sum()), "fallbacks", flush=True)
    np.savez_compressed(T.GOLDEN, **out)
    print("wrote", T.GOLDEN)


if __name__ == "__main__":
    main()
