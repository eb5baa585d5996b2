"""Who frees and counts device memory (nudge_b200/csrc/nb_api.cu, DevBuf and alloc_zeroed), with nb_debug_read("device_bytes") as the
measure: a shard's buffers are its own, counted while it exists and returned by nb_shard_destroy; a failed nb_shard_create leaves no shard,
no bytes and no sharded context behind; and a table created on first use is allocated and counted once."""
import ctypes
import numpy as np
import pytest
import nudge_b200
from nudge_b200 import abi, scenes
from tests.gpu_util import side_stream
from tests.test_gpu_buffers import device_bytes

pytestmark = pytest.mark.gpu

NB_ERR_CUDA = -1
INBOX_BYTES_PER_GHOST = 16 * 2 * 2 * (1 + 24)   # the per-sweep inbox and the pass-indexed one of 24 passes (nb_shard_api.cuh)


def _scene():
    return scenes.demo_scene(300, 300, iterations=4, spread=8.0, height=12.0, seed=47)


def test_shard_buffers_are_counted_and_freed_by_its_destroy():
    s = _scene()
    x = nudge_b200.Sim(s, stream=side_stream())
    before = device_bytes(x)
    ghosts = 4096
    x.shard_create(0, 1, None, ghosts, 1024)
    assert device_bytes(x) >= before + INBOX_BYTES_PER_GHOST * ghosts
    x.lib.nb_shard_destroy(x.shard)
    x.shard = None
    assert device_bytes(x) == before
    x.close()


def test_failed_shard_create_leaves_nothing_behind():
    s = _scene()
    x = nudge_b200.Sim(s, stream=side_stream(), max_bodies=s.n_bodies + 4, max_boxes=s.n_boxes + 4)
    before = device_bytes(x)
    out = ctypes.c_void_p(1)   # overwritten with null
    r = x.lib.nb_shard_create(x.ctx, 0, 1, None, 0xffffffff, 64, ctypes.byref(out))   # an inbox of about 6.9 TB: no device holds it
    assert r == NB_ERR_CUDA
    assert "cudaMalloc" in x.lib.nb_last_error(x.ctx).decode()
    assert out.value is None
    assert device_bytes(x) == before
    # the context is not sharded: an edit is accepted
    fr = scenes.fragment(np.array([[0.0, 20.0, 0.0], [3.0, 20.0, 0.0]]), first_tag=int(max(s.box_tags.max(), s.sphere_tags.max())) + 1)
    x.add_bodies(fr)
    assert x.scene.n_bodies == s.n_bodies + 2
    x.close()


def _rays(n):
    r = np.zeros(n, abi.RAY)
    r["origin"] = (0.0, 30.0, 0.0); r["direction"] = (0.0, -1.0, 0.0); r["max_t"] = 100.0
    r["mask"] = 0xffffffff; r["ignore_body"] = abi.RAY_NO_HIT
    return r


def _enable_debug(x):
    x._ck(x.lib.nb_debug_enable(x.ctx, 1), "nb_debug_enable")


# name -> a call that creates its table on first use (plus, for the calls with host staging, buffers grown to the call's size)
FIRST_USE = {
    "kind": lambda x: x.upload_kinematic_bodies(np.array([(1, (0.0, 0.5, 0.0), (0.0, 0.0, 0.0), 0)], scenes.KINEMATIC)),
    "body_forces": lambda x: x.set_body_forces(scenes.default_body_forces(np.arange(1, 17, dtype=np.uint32))),
    "impulse_sort": lambda x: x.apply_body_impulses(np.array([(3, (0.0, 0.0, 0.0), (0.0, 1.0, 0.0), (0.0, 0.0, 0.0), (0, 0))], scenes.BODY_IMPULSE)),
    "instance_matrices": lambda x: x.instance_matrices(),
    "debug_pair_keys": _enable_debug,
    "ray_scratch": lambda x: x.raycast(_rays(64)),
}


@pytest.mark.parametrize("name", sorted(FIRST_USE))
def test_table_created_on_first_use_is_counted_once(name):
    call = FIRST_USE[name]
    x = nudge_b200.Sim(_scene(), stream=side_stream())
    before = device_bytes(x)
    call(x)
    first = device_bytes(x)
    assert first > before, name
    call(x)
    assert device_bytes(x) == first, name
    x.close()
