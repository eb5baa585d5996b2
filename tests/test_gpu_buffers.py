"""The editing calls' device buffers and host staging (nudge_b200/csrc/nb_api.cu, DevBuf / grow / put_staged): a buffer grown in steps holds
what one call at the final size holds, with nb_debug_read("device_bytes") as the measure, for every buffer an editing call grows; a snapshot's
bytes go with nb_snapshot_destroy; and the caller's array may be overwritten as soon as the call returns, pinned or not, while the copy is
still queued behind earlier steps."""
import ctypes
import numpy as np
import pytest
import nudge_b200
from nudge_b200 import abi, scenes
from tests.gpu_util import side_stream

pytestmark = pytest.mark.gpu


def _scene():
    return scenes.demo_scene(1500, 1500, iterations=8, spread=8.0, height=14.0, seed=41)


def _sim(s, **kw):
    return nudge_b200.Sim(s, stream=side_stream(), **kw)


def device_bytes(x):
    v = np.zeros(1, np.uint64)
    n = ctypes.c_size_t(0)
    x._ck(x.lib.nb_debug_read(x.ctx, b"device_bytes", abi.ptr(v), 8, ctypes.byref(n), x.stream), "nb_debug_read")
    assert n.value == 8
    return int(v[0])


def _rows(n, B):
    r = np.zeros(n, nudge_b200.ROW)
    r["a"] = 1 + np.arange(n) % (B - 1); r["lin_a"][:, 1] = 1.0; r["lo"] = -1.0; r["hi"] = 1.0
    return r


def _kinematic(n):
    k = np.zeros(n, scenes.KINEMATIC)
    k["body"] = 1 + np.arange(n); k["velocity"][:, 1] = 0.5
    return k


def _impulses(n, B):
    e = np.zeros(n, scenes.BODY_IMPULSE)
    e["body"] = 1 + np.arange(n) % (B - 1); e["impulse"][:, 1] = 0.25   # a body may be listed again
    return e


def _forces(n):
    f = scenes.default_body_forces(1 + np.arange(n))
    f["gravity_scale"] = 0.5
    return f


def _sensor_flags(s):
    f = np.zeros(s.n_colliders, np.uint8)
    f[::10] = 1
    return f


# name -> (sizes, call(sim, size)); each call grows one buffer (or, for the snapshot rows, the user rows and the snapshot's copy of them)
GROWN = {
    "constraint_rows": ((64, 512, 4096, 16384), lambda x, n: x.upload_constraint_rows(_rows(n, x.scene.n_bodies))),
    "kinematic": ((16, 256, 2048), lambda x, n: x.upload_kinematic_bodies(_kinematic(n))),
    "impulses": ((16, 512, 8192), lambda x, n: x.apply_body_impulses(_impulses(n, x.scene.n_bodies))),
    "forces": ((16, 256, 2048), lambda x, n: x.set_body_forces(_forces(n))),
    "remove": ((16, 128, 1024), lambda x, n: x.remove_bodies(1 + np.arange(n))),
    "contact_events": ((64, 4096, 65536), lambda x, n: x.enable_contact_events(n)),
    "sensor_pairs": ((1024, 8192, 65536), lambda x, n: x.upload_sensors(_sensor_flags(x.scene), max_pairs=n)),
}


@pytest.mark.parametrize("name", sorted(GROWN))
def test_growing_in_steps_holds_what_growing_once_holds(name):
    sizes, call = GROWN[name]
    s = _scene()
    a, b = _sim(s), _sim(s)
    assert device_bytes(a) == device_bytes(b)
    for n in sizes:
        call(a, n)
    call(b, sizes[-1])
    assert device_bytes(a) == device_bytes(b), name


def test_snapshot_rows_grown_by_saves_and_user_rows_grown_by_a_restore():
    s = _scene()
    B = s.n_bodies
    # snapshot rows: saves of a growing row set into one snapshot hold what one save of the final set holds
    a, b = _sim(s), _sim(s)
    snap_a = None
    for n in (64, 512, 4096):
        a.upload_constraint_rows(_rows(n, B))
        snap_a = a.snapshot(into=snap_a)
    b.upload_constraint_rows(_rows(4096, B))
    snap_b = b.snapshot()
    assert device_bytes(a) == device_bytes(b)
    # user rows through a restore: back from 64 rows to a snapshot of 4096 holds what the 4096 rows held
    c, d = _sim(s), _sim(s)
    c.upload_constraint_rows(_rows(64, B))
    snap_c = c.snapshot()
    c.upload_constraint_rows(_rows(4096, B))
    c.snapshot(into=snap_c)
    c.upload_constraint_rows(_rows(64, B))
    c.restore(snap_c)
    d.upload_constraint_rows(_rows(4096, B))
    snap_d = d.snapshot()
    d.restore(snap_d)
    assert device_bytes(c) == device_bytes(d)
    assert np.array_equal(c.download_constraint_rows(4096), d.download_constraint_rows(4096))


def test_snapshot_destroy_returns_its_bytes():
    s = _scene()
    x = _sim(s)
    x.upload_sensors(_sensor_flags(s))
    x.upload_constraint_rows(_rows(3000, s.n_bodies))
    x.upload_constraint_rows(_rows(1000, s.n_bodies))   # the context's rows keep room for 3000
    before = device_bytes(x)
    snap = x.snapshot()   # the arena, and the rows and the overlap list sized by the save
    x.upload_constraint_rows(_rows(3000, s.n_bodies))
    x.snapshot(into=snap)   # the snapshot's rows grow; the context's do not
    assert device_bytes(x) > before + 3000 * nudge_b200.ROW.itemsize
    snap.close()
    assert device_bytes(x) == before


def _pinned(a, keep):
    """A copy of `a` in page-locked host memory, whose copies cudaMemcpyAsync runs in stream order; `keep` holds the allocation."""
    import torch
    t = torch.empty(max(a.nbytes, 1), dtype=torch.uint8, pin_memory=True)
    keep.append(t)
    v = t.numpy()[:a.nbytes].view(a.dtype)
    v[:] = a
    return v


def _busy(x, steps=200):
    """Steps queued on x's stream (200 of this scene take about 0.3 s on an H100 at 700 W): a copy queued after them cannot start before
    they end."""
    for _ in range(3):
        x.step()
    x.download_bodies()   # the step graph is recorded
    for _ in range(steps):
        x.step()


def _call(x, fn, rows):
    x._ck(getattr(x.lib, fn)(x.ctx, abi.ptr(rows), len(rows), x.stream), fn)


# Each test makes a first call with the same list before the steps are queued, so that the call under test grows no buffer (a growth
# synchronises the stream, after which even an unstaged copy would run at once).

def test_kinematic_rows_may_be_reused_on_return_pinned():
    s, keep = _scene(), []
    x = _sim(s)
    first = _kinematic(64)
    first["velocity"][:, 0] = np.arange(64, dtype=np.float32)
    rows = _pinned(first, keep)
    x.upload_kinematic_bodies(first)
    _busy(x)
    _call(x, "nb_upload_kinematic_bodies", rows)
    rows["velocity"] = (-7.0, 1.0, 2.0)
    x.download_bodies()
    assert np.array_equal(x.momentum["velocity"][first["body"]], first["velocity"])


def test_impulse_rows_may_be_reused_on_return_pinned():
    s, keep = _scene(), []
    x = _sim(s)
    first = _impulses(300, s.n_bodies)
    first["impulse"][:, 0] = np.linspace(-2.0, 2.0, 300, dtype=np.float32)
    rows = _pinned(first, keep)
    x.apply_body_impulses(first)
    _busy(x)
    zero = np.zeros(s.n_bodies, scenes.MOMENTUM)   # the momentum the impulses land on
    x._ck(x.lib.nb_upload_momentum(x.ctx, abi.ptr(zero), len(zero), x.stream), "nb_upload_momentum")
    _call(x, "nb_apply_body_impulses", rows)
    rows["impulse"] = (0.0, 50.0, 0.0)
    want = zero.copy()
    b = first["body"].astype(np.int64)
    want["velocity"][b] = s.properties["mass_inverse"][b, None] * first["impulse"]   # float32, as the kernel computes it
    x.download_bodies()
    assert x.momentum.tobytes() == want.tobytes()


def test_force_rows_may_be_reused_on_return_pinned():
    s, keep = _scene(), []
    x = _sim(s)
    first = _forces(500)
    first["force"][:, 1] = np.arange(500, dtype=np.float32)
    first["reserved"] = 7   # stored as 0
    rows = _pinned(first, keep)
    x.set_body_forces(first)
    _busy(x)
    _call(x, "nb_set_body_forces", rows)
    rows["gravity_scale"] = 3.0; rows["force"] = 0.0
    want = first.copy()
    want["reserved"] = 0
    assert x.download_body_forces()[first["body"]].tobytes() == want.tobytes()


def test_added_body_and_collider_arrays_may_be_reused_on_return_pinned():
    s, keep = _scene(), []
    B, n = s.n_bodies, 40
    x = _sim(s, max_bodies=B + n, max_boxes=s.n_boxes + n)
    fr = scenes.fragment(np.stack([np.arange(n), np.full(n, 30.0), np.zeros(n)], 1) * 1.5, first_tag=int(max(s.box_tags.max(), s.sphere_tags.max())) + 1)
    fr.momentum["velocity"][:, 2] = np.arange(n, dtype=np.float32); fr.idle[:] = 3
    bx = fr.box_transforms.copy()
    bx["body"] += np.uint32(B)
    first = dict(transforms=fr.transforms, properties=fr.properties, momentum=fr.momentum, idle=fr.idle, box_tags=fr.box_tags, box_data=fr.box_data,
                 box_transforms=bx)
    p = {k: _pinned(v, keep) for k, v in first.items()}
    P = abi.ptr
    bodies = abi.BodyData(P(p["transforms"]), P(p["properties"]), P(p["momentum"]), P(p["idle"]), n)
    cols = abi.ColliderData(abi.Shapes(P(p["box_tags"]), P(p["box_data"]), P(p["box_transforms"]), n), abi.Shapes(None, None, None, 0))
    _busy(x)
    x._ck(x.lib.nb_add_bodies(x.ctx, ctypes.byref(bodies), ctypes.byref(cols), None, x.stream), "nb_add_bodies")
    p["transforms"]["position"] += 100.0; p["properties"]["mass_inverse"] = 2.0; p["momentum"]["velocity"] = 5.0; p["idle"][:] = 0
    p["box_tags"] += np.uint32(n); p["box_data"]["size"] = 0.75; p["box_transforms"]["position"] = 1.0
    out = {k: abi.aligned_array(B + n, dt) for k, dt in (("transforms", scenes.TRANSFORM), ("properties", scenes.PROPERTIES),
                                                           ("momentum", scenes.MOMENTUM), ("idle", np.uint8))}
    h = abi.BodyData(P(out["transforms"]), P(out["properties"]), P(out["momentum"]), P(out["idle"]), B + n)
    x._ck(x.lib.nb_download_bodies(x.ctx, ctypes.byref(h), x.stream), "nb_download_bodies")
    for k in ("transforms", "momentum", "idle"):
        assert out[k][B:].tobytes() == first[k].tobytes(), k
    c = x.download_colliders()
    for k in ("box_tags", "box_data", "box_transforms"):
        assert c[k][-n:].tobytes() == first[k].tobytes(), k
