"""The solver's per-body chains (k_batch_index counts, k_chain_alloc / k_chain_scatter / k_chain_rank) against the definition they
replace: a stable sort of the (body | batch) keys of the entries e = 2*i + side, whose position inside a body's run is `seq` and
whose run length is `len` (rows.wait = (seq, len); static-world sides get (0, 0))."""
import numpy as np
import pytest
import nudge_b200
from nudge_b200 import scenes

pytestmark = pytest.mark.gpu


def _expected_waits(g):
    g.download_contacts()
    n = int(g.counts().contacts)
    sorted_ = g.debug("sorted", np.uint32)[:n]
    batch = g.debug("batch_of", np.uint32)[:n].astype(np.int64)
    slot = g.debug("slot_idx", np.uint32)[:n].astype(np.int64)
    stride = g.debug_scalar("row_stride")
    ab = g.contact_bodies[:n][sorted_]
    body = np.stack([ab["a"], ab["b"]], axis=1).reshape(-1).astype(np.int64)   # entry e = 2*i + side
    bat = np.repeat(batch, 2)
    e = np.arange(2 * n)
    order = np.lexsort((e, bat, body))          # the stable sort on (body, batch) over entry order
    sb = body[order]
    first = np.r_[True, sb[1:] != sb[:-1]]
    run_start = np.maximum.accumulate(np.where(first, np.arange(2 * n), 0))
    seq = np.empty(2 * n, np.int64); seq[order] = np.arange(2 * n) - run_start
    length = np.bincount(body, minlength=int(body.max()) + 1 if n else 1)[body]
    real = body != 0
    want = np.zeros((2, stride, 2), np.uint32)
    side = e & 1
    s = np.repeat(slot, 2)
    want[side[real], s[real], 0] = seq[real]
    want[side[real], s[real], 1] = length[real]
    got = g.debug("row_wait", np.uint32).reshape(2, stride, 2)
    used = np.zeros((2, stride), bool); used[side, s] = True
    return got, want, used, length[real].max() if real.any() else 0


@pytest.mark.parametrize("name,make,steps", [
    ("hub_inside_the_on_chip_list", lambda: scenes.hub_platform(12, iterations=4), 2),
    ("hub_spilling_the_list", lambda: scenes.hub_platform(55, iterations=4), 1),
    ("pile", lambda: scenes.box_drop(6000, iterations=8, seed=3), 120),
    ("mixed", lambda: scenes.demo_scene(400, 400, iterations=4, spread=2.0, height=20.0), 60),
])
def test_chain_ranks_equal_the_stable_sort(name, make, steps):
    g = nudge_b200.Sim(make(), debug=True)
    for _ in range(steps):
        g.step_staged()
    assert g.counts().overflow == 0
    got, want, used, longest = _expected_waits(g)
    assert used.any()
    assert np.array_equal(got[used], want[used]), name
    if name.startswith("hub"):
        assert longest > 300          # one long chain, handled by the same kernels


def test_chain_ranks_stay_right_step_after_step():
    """The counts, segment cursors and segments are rebuilt every step: nothing of the previous step's chains may leak into the next."""
    s = scenes.demo_scene(40, 40, iterations=4, spread=2.0, height=4.0, seed=4)
    g = nudge_b200.Sim(s, contact_capacity=20000, debug=True)
    for _ in range(30):
        g.step_staged()
        assert g.counts().overflow == 0
        got, want, used, _ = _expected_waits(g)
        assert np.array_equal(got[used], want[used])
