"""nb_get_body_states / nb_set_body_states (DESIGN.md section 8.19): nb_launch_count's delta over a torch.profiler window of each call, in
host and device mode, equals the header's launch count and the number of this library's kernel records in the window.  A file of its own,
run after test_gpu_launch_count.py: a profiler session can leave the driver's memset records of later work to the next session."""
import numpy as np
import pytest
import torch
import nudge_b200
from nudge_b200 import abi, scenes
from tests.gpu_util import side_stream
from tests.test_gpu_launch_count import LIBRARY_KERNEL, _window
from tests.test_gpu_body_states import _random_rows

pytestmark = pytest.mark.gpu
POSE, VEL = abi.BODY_POSE, abi.BODY_VELOCITY


def test_launch_counts_equal_the_profiler_and_the_header(tmp_path):
    s = scenes.demo_scene(400, 400, iterations=4, spread=6.0, height=10.0, seed=7)
    g = nudge_b200.Sim(s, stream=side_stream())
    g.step(); g.step()
    rows = _random_rows(np.random.default_rng(8), s.n_bodies, 40)
    idx = rows["body"].copy()
    t_rows = torch.from_numpy(rows.view(np.int32).reshape(-1).copy()).cuda()
    t_idx = torch.from_numpy(idx.view(np.int32)).cuda()
    t_out = torch.zeros(len(idx) * 16, dtype=torch.int32, device="cuda")
    g.set_body_states(rows, POSE)   # allocates the set's scratch outside the windows
    torch.cuda.synchronize()
    cases = [(lambda: g.get_body_states(idx), 1), (lambda: g.get_body_states(device_ptrs=(t_idx.data_ptr(), t_out.data_ptr()), n=len(idx)), 1),
             (lambda: g.set_body_states(rows, VEL), 3), (lambda: g.set_body_states(rows, POSE), 6), (lambda: g.set_body_states(rows, POSE | VEL), 6),
             (lambda: g.set_body_states(None, VEL, device_ptrs=(t_rows.data_ptr(), 0), n=len(rows)), 3),
             (lambda: g.set_body_states(None, POSE | VEL, device_ptrs=(t_rows.data_ptr(), 0), n=len(rows)), 6),
             (lambda: g.step(), 61)]
    for k, (calls, want) in enumerate(cases):
        counted, names = _window(g, calls, tmp_path)
        # the records are this library's kernels, and at most the driver's own kernels of a cudaMemsetAsync (the pose set clears its byte per body)
        assert [n for n in names if not LIBRARY_KERNEL.match(n) and not n.startswith("memset")] == [], k
        assert counted == want == len([n for n in names if LIBRARY_KERNEL.match(n)]), (k, counted, want, names)
