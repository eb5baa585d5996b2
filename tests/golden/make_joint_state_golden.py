"""Records tests/golden/joint_state.npz: the scene of tests/test_gpu_joint_state_golden.py (every joint table, a continuous-collision set,
kinematic bodies, body forces, filters and sensors, parity mode) saved to a state file after 20 steps, and a fresh context that loads the
file and steps 20 more times.  Needs a GPU and the built library; records what this tree's build computes.

    python tests/golden/make_joint_state_golden.py"""
import os, sys, tempfile
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from tests import test_gpu_joint_state_golden as T  # noqa: E402


def main(out=T.GOLDEN):
    with tempfile.TemporaryDirectory() as d:
        rec = T.record(d)
    np.savez_compressed(out, **rec)
    print("wrote", out, {k: len(v) for k, v in rec.items()})


if __name__ == "__main__":
    main(*sys.argv[1:])
