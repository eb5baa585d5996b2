"""A joint set through a state file against a committed recording (tests/golden/joint_state.npz, made by
tests/golden/make_joint_state_golden.py): a seeded small pile in parity mode with joints of all four types, drives with every flag (some
broken), springs on each type, a continuous-collision set, a kinematic body, body forces, filters and sensors.  The bytes of nb_save_state's
file after 20 steps, then the bodies, joints, drives and springs of a fresh context that loads the file and steps 20 more times, must equal
the recording byte for byte.  The save comes after steps because a load followed by a save is not byte-stable: drive and spring positions
are rewritten only by the next row build."""
import os
import numpy as np
import pytest
import nudge_b200
from nudge_b200 import scenes
from oracle import joints_ref
from tests.test_gpu_joints import _joints_at_rest, _body_bytes
from tests.test_gpu_joint_dof import _random_drives
from tests.test_gpu_joint_springs import _random_springs

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "joint_state.npz")
STEPS = 20
ALL_FLAGS = 0x77   # LIMIT | MOTOR | BREAKABLE | SLIDE | CONE | TWIST


def _scene():
    s = scenes.demo_scene(60, 60, iterations=4, seed=11, spread=3.0, height=8.0)
    rng = np.random.default_rng(11)
    K = s.n_colliders
    s.sensors = np.zeros(K, np.uint8); s.sensors[[3, 70]] = 1
    s.collision_filters = np.zeros(K, scenes.FILTER)
    s.collision_filters["category"] = 1 << rng.integers(0, 3, K)
    s.collision_filters["mask"] = np.where(rng.random(K) < 0.1, 0xfffe, 0xffff)
    s.filter_flags = scenes.FILTER_SKIP_CONNECTED
    s.connections = np.array([(5, 6), (20, 21)], scenes.PAIR32)
    s.kinematic = np.array([(9, (0.5, 0.0, 0.0), (0.0, 0.3, 0.0), 0)], scenes.KINEMATIC)
    f = scenes.default_body_forces(np.arange(30, 50))
    f["gravity_scale"] = rng.uniform(0.0, 2.0, len(f)).astype(np.float32)
    f["linear_damping"] = rng.uniform(0.0, 0.5, len(f)).astype(np.float32)
    s.body_forces = f
    return s


def build_sim():
    """The seeded scene with every joint table, a continuous-collision set and the other tables uploaded, in parity mode."""
    s = _scene()
    g = nudge_b200.Sim(s)
    g.set_solver_mode("parity")
    rng = np.random.default_rng(5)
    joints = _joints_at_rest(s.transforms, rng, 48, s.n_bodies)
    drives = _random_drives(joints, rng, share=0.9, broken=0.15, fragile=0.1)
    springs = _random_springs(joints, rng, share=0.7)
    g.upload_joints(joints); g.upload_joint_drives(drives); g.upload_joint_springs(springs)
    g.upload_ccd_bodies([(b, 0.2, 0.1, 0xffff, 0xffff) for b in (12, 40, 77)])
    types = joints["type"]
    assert set(types.tolist()) == {joints_ref.BALL, joints_ref.HINGE, joints_ref.FIXED, joints_ref.DISTANCE}
    assert np.bitwise_or.reduce(drives["flags"]) == ALL_FLAGS and drives["broken"].any()
    assert set(types[springs["joint"]].tolist()) == set(types.tolist())
    return s, g


def record(tmp_dir):
    """The file's bytes after STEPS steps, then the state of a fresh context that loaded it after STEPS more."""
    s, g = build_sim()
    for _ in range(STEPS):
        g.step()
    path = os.path.join(tmp_dir, "joints.nbstate")
    g.save_state(path)
    with open(path, "rb") as fh:
        state = fh.read()
    h = nudge_b200.Sim(s)
    h.load_state(path)
    for _ in range(STEPS):
        h.step()
    out = {"state": state, "bodies": _body_bytes(h), "joints": h.download_joints().tobytes(),
           "drives": h.download_joint_drives().tobytes(), "springs": h.download_joint_springs().tobytes()}
    return {k: np.frombuffer(v, np.uint8) for k, v in out.items()}


@pytest.mark.gpu
def test_state_file_and_its_load_equal_the_recording(tmp_path):
    want = np.load(GOLDEN)
    got = record(str(tmp_path))
    assert int.from_bytes(got["state"][8:12].tobytes(), "little") == 9
    for k in ("state", "bodies", "joints", "drives", "springs"):
        assert got[k].tobytes() == want[k].tobytes(), k
