"""Device tables allocated on first use (the body-force table, the kinematic table) are zeroed before the first kernel that fills them, also
when that kernel runs on a non-blocking stream while the legacy default stream still holds another context's step: the zero fill must not
land after the fill (it did, now and then: a fresh body-force table read all zeros, every gravity scale 0)."""
import numpy as np
import pytest
import nudge_b200
from nudge_b200 import scenes
from tests.gpu_util import side_stream

pytestmark = pytest.mark.gpu


def test_tables_created_on_a_side_stream_right_after_a_step_on_the_legacy_stream():
    import torch
    s = scenes.demo_scene(300, 300, iterations=4, spread=12.0, height=20.0, seed=43)
    rows = scenes.default_body_forces(np.arange(1, s.n_bodies, dtype=np.uint32))
    rows["gravity_scale"] = 0.5
    k = s.n_bodies - 1
    for rep in range(30):
        a, b = nudge_b200.Sim(s, stream=side_stream(), debug=True), nudge_b200.Sim(s)   # b: the legacy default stream
        a.step(); b.step()
        a.set_body_forces(rows)   # allocates the table
        b.step()
        a.upload_kinematic_bodies(np.array([(k, (0.0, 1.0, 0.0), (0.0, 0.0, 0.0), 0)], scenes.KINEMATIC))   # allocates the kind table
        torch.cuda.synchronize()
        got = a.download_body_forces()
        assert (got["gravity_scale"][1:] == np.float32(0.5)).all() and (got["body"] == np.arange(s.n_bodies)).all(), rep
        assert a.debug("kind", np.uint8)[k] & 1, rep
        a.close(); b.close()
