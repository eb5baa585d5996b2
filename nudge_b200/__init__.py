"""nudge_b200 — H100-native (sm_90a) rigid-body simulation step, drop-in for rasmusbarr/nudge's hot path.

This package is only the Python binding used by tests and bench.py: it loads the C-ABI shared library
(include/nudge_b200.h, built by nudge_b200/csrc/build.sh) with ctypes and mirrors the reference's seven calls
(nudge.h:134-146) on a device-resident simulation.  There is no CPU path: importing works without a GPU
(so the symbol check can run), creating a `Sim` does not."""
import ctypes as C
import os
import numpy as np
from . import abi, scenes

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "lib", "libnudge_b200.so")

EXPORTS = ["nb_create", "nb_destroy", "nb_last_error", "nb_upload_bodies", "nb_upload_colliders", "nb_upload_connections", "nb_upload_cache",
           "nb_upload_contacts", "nb_download_bodies", "nb_download_contacts", "nb_download_cache", "nb_download_counts", "nb_upload_momentum", "nb_upload_transforms",
           "nb_download_momentum", "nb_download_transforms", "nb_collide", "nb_apply_gravity_damping", "nb_read_cached_impulses",
           "nb_setup_contact_constraints", "nb_apply_impulses", "nb_update_cached_impulses", "nb_write_cached_impulses", "nb_advance", "nb_step",
           "nb_launch_count", "nb_debug_read", "nb_debug_rcp", "nb_lut_model_exact", "nb_debug_sort", "nb_debug_scan", "nb_debug_enable", "nb_pack_momentum", "nb_unpack_momentum",
           "nb_shard_unique_id", "nb_shard_create", "nb_shard_destroy", "nb_shard_ipc_handle", "nb_shard_open_peer", "nb_shard_plan", "nb_shard_exchange",
           "nb_shard_step", "nb_shard_graph_active", "nb_shard_partition", "nb_shard_debug_no_exchange",
           "nb_set_solver_mode", "nb_get_solver_mode", "nb_debug_timing_enable", "nb_debug_timing",
           "nb_stream_create", "nb_stream_destroy", "nb_stream_synchronize", "nb_save_state", "nb_load_state", "nb_state_info",
           "nb_upload_constraint_rows", "nb_download_constraint_rows", "nb_instance_matrices", "nb_shard_build_plan", "nb_shard_local_scene",
           "nb_enable_contact_events", "nb_download_contact_events", "nb_upload_collision_filters",
           "nb_upload_sensors", "nb_download_sensor_overlaps", "nb_upload_kinematic_bodies", "nb_apply_body_impulses", "nb_apply_radial_impulse",
           "nb_add_bodies", "nb_remove_bodies", "nb_download_colliders", "nb_download_connections",
           "nb_set_body_forces", "nb_clear_body_forces", "nb_download_body_forces",
           "nb_snapshot_create", "nb_snapshot_destroy", "nb_snapshot_save", "nb_snapshot_restore", "nb_upload_joints", "nb_download_joints", "nb_raycast", "nb_overlap",
           "nb_shapecast", "nb_upload_joint_drives", "nb_download_joint_drives", "nb_get_body_states", "nb_set_body_states",
           "nb_upload_joint_springs", "nb_download_joint_springs", "nb_get_body_contact_impulses", "nb_get_contact_pair_impulses"]


class Config(C.Structure):
    _fields_ = [("max_bodies", C.c_uint32), ("max_boxes", C.c_uint32), ("max_spheres", C.c_uint32), ("max_connections", C.c_uint32),
                ("max_pairs", C.c_uint32), ("max_contacts", C.c_uint32), ("device", C.c_int)]


class Counts(C.Structure):
    _fields_ = [(n, C.c_uint32) for n in ("pairs", "live_pairs", "contacts", "sleeping", "active", "cache", "culled", "batches", "levels", "overflow")]


_lib = None


def load_library():
    """Loads the CUDA extension; raises if it has not been built (there is no fallback)."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError("nudge_b200: %s is missing — run nudge_b200/csrc/build.sh (or __graft_entry__.build()); there is no CPU path" % LIB_PATH)
        lib = C.CDLL(LIB_PATH)
        V = C.c_void_p
        lib.nb_create.argtypes = [V, V]
        lib.nb_destroy.argtypes = [V]
        lib.nb_last_error.argtypes = [V]; lib.nb_last_error.restype = C.c_char_p
        for f in ("nb_upload_bodies", "nb_upload_colliders", "nb_upload_connections", "nb_upload_cache", "nb_download_bodies", "nb_download_cache", "nb_download_counts"):
            getattr(lib, f).argtypes = [V, V, V]
        lib.nb_download_contacts.argtypes = [V, V, V, V]
        lib.nb_upload_contacts.argtypes = [V, V, V, V]
        for f in ("nb_upload_momentum", "nb_upload_transforms", "nb_download_momentum", "nb_download_transforms"):
            getattr(lib, f).argtypes = [V, V, C.c_uint32, V]
        for f in ("nb_collide", "nb_read_cached_impulses", "nb_setup_contact_constraints", "nb_update_cached_impulses", "nb_write_cached_impulses"):
            getattr(lib, f).argtypes = [V, V]
        lib.nb_apply_gravity_damping.argtypes = [V, C.c_float, C.c_float, C.c_float, V]
        lib.nb_apply_impulses.argtypes = [V, C.c_uint32, V]
        lib.nb_advance.argtypes = [V, C.c_float, V]
        lib.nb_step.argtypes = [V, C.c_float, C.c_uint32, C.c_float, C.c_float, V]
        lib.nb_launch_count.argtypes = [V]; lib.nb_launch_count.restype = C.c_uint64
        lib.nb_debug_read.argtypes = [V, C.c_char_p, V, C.c_size_t, V, V]
        lib.nb_debug_rcp.argtypes = [V, V, V, C.c_uint32, C.c_int]
        lib.nb_lut_model_exact.argtypes = [V]
        lib.nb_debug_sort.argtypes = [V, V, V, C.c_uint32, C.c_int, C.c_int]
        lib.nb_debug_scan.argtypes = [V, V, C.c_uint32, V]
        lib.nb_debug_enable.argtypes = [V, C.c_int]
        lib.nb_pack_momentum.argtypes = [V, V, C.c_uint32, V, V]
        lib.nb_unpack_momentum.argtypes = [V, V, V, C.c_uint32, V, V]
        lib.nb_shard_unique_id.argtypes = [V]
        lib.nb_shard_create.argtypes = [V, C.c_uint32, C.c_uint32, V, C.c_uint32, C.c_uint32, V]
        lib.nb_shard_destroy.argtypes = [V]; lib.nb_shard_destroy.restype = None
        lib.nb_shard_ipc_handle.argtypes = [V, V]
        lib.nb_shard_open_peer.argtypes = [V, C.c_uint32, V]
        lib.nb_shard_plan.argtypes = [V, V, C.c_uint32, V, V, V, V, V, C.c_uint32, C.c_uint32, V]
        lib.nb_shard_exchange.argtypes = [V, C.c_int, V]
        lib.nb_shard_step.argtypes = [V, C.c_float, C.c_uint32, C.c_float, C.c_float, C.c_int, V]
        lib.nb_shard_graph_active.argtypes = [V]
        lib.nb_shard_debug_no_exchange.argtypes = [V, C.c_int]
        lib.nb_shard_partition.argtypes = [V, V, C.c_uint32, C.c_uint32, C.c_uint32, C.c_float, C.c_uint32, V, V, V, C.c_uint32]
        lib.nb_set_solver_mode.argtypes = [V, C.c_int]
        lib.nb_get_solver_mode.argtypes = [V]
        lib.nb_debug_timing_enable.argtypes = [V, C.c_int]
        lib.nb_debug_timing.argtypes = [V, V, V, V]
        lib.nb_stream_create.argtypes = [V]; lib.nb_stream_create.restype = V
        lib.nb_stream_destroy.argtypes = [V, V]; lib.nb_stream_destroy.restype = None
        lib.nb_stream_synchronize.argtypes = [V, V]
        lib.nb_save_state.argtypes = [V, C.c_char_p, V]
        lib.nb_load_state.argtypes = [V, C.c_char_p, V]
        lib.nb_state_info.argtypes = [C.c_char_p, V]
        lib.nb_upload_constraint_rows.argtypes = [V, V, C.c_uint32, V]
        lib.nb_download_constraint_rows.argtypes = [V, V, C.c_uint32, V]
        lib.nb_upload_joints.argtypes = [V, V, C.c_uint32, V]
        lib.nb_download_joints.argtypes = [V, V, C.c_uint32, V, V]
        lib.nb_upload_joint_drives.argtypes = [V, V, C.c_uint32, V]
        lib.nb_download_joint_drives.argtypes = [V, V, C.c_uint32, V, V]
        lib.nb_upload_joint_springs.argtypes = [V, V, C.c_uint32, V]
        lib.nb_download_joint_springs.argtypes = [V, V, C.c_uint32, V, V]
        lib.nb_instance_matrices.argtypes = [V, V, C.c_uint32, C.c_int, V, V]
        lib.nb_shard_build_plan.argtypes = [V, C.c_uint32, V, V, C.c_uint32, C.c_uint32, V, V, V, V, V, V, V, V]
        lib.nb_shard_local_scene.argtypes = [V, C.c_uint32, V, C.c_uint32, C.c_uint32, V, C.c_uint32, V, C.c_uint32, V, V, V, V, V]
        lib.nb_enable_contact_events.argtypes = [V, C.c_uint32]
        lib.nb_download_contact_events.argtypes = [V, V, C.c_uint32, V, V, V]
        lib.nb_upload_collision_filters.argtypes = [V, V, C.c_uint32, C.c_uint32, V]
        lib.nb_upload_sensors.argtypes = [V, V, C.c_uint32, C.c_uint32, V]
        lib.nb_download_sensor_overlaps.argtypes = [V, V, C.c_uint32, V, V]
        lib.nb_upload_kinematic_bodies.argtypes = [V, V, C.c_uint32, V]
        lib.nb_apply_body_impulses.argtypes = [V, V, C.c_uint32, V]
        lib.nb_apply_radial_impulse.argtypes = [V, V, V]
        lib.nb_add_bodies.argtypes = [V, V, V, V, V]
        lib.nb_remove_bodies.argtypes = [V, V, C.c_uint32, V]
        lib.nb_download_colliders.argtypes = [V, V, V]
        lib.nb_download_connections.argtypes = [V, V, C.c_uint32, V]
        lib.nb_set_body_forces.argtypes = [V, V, C.c_uint32, V]
        lib.nb_clear_body_forces.argtypes = [V, V]
        lib.nb_download_body_forces.argtypes = [V, V, C.c_uint32, V, V]
        lib.nb_snapshot_create.argtypes = [V, V]
        lib.nb_snapshot_destroy.argtypes = [V]; lib.nb_snapshot_destroy.restype = None
        lib.nb_snapshot_save.argtypes = [V, V, V]
        lib.nb_snapshot_restore.argtypes = [V, V, V]
        lib.nb_raycast.argtypes = [V, V, C.c_uint32, V, C.c_uint32, C.c_int, V]
        lib.nb_overlap.argtypes = [V, V, C.c_uint32, V, C.c_uint32, V, C.c_uint32, C.c_int, V]
        lib.nb_shapecast.argtypes = [V, V, C.c_uint32, V, C.c_uint32, C.c_int, V]
        lib.nb_upload_ccd_bodies.argtypes = [V, V, C.c_uint32, V]
        lib.nb_download_ccd_bodies.argtypes = [V, V, C.c_uint32, V, V]
        lib.nb_get_body_states.argtypes = [V, V, C.c_uint32, V, C.c_int, V]
        lib.nb_set_body_states.argtypes = [V, V, C.c_uint32, C.c_uint32, V, C.c_int, V]
        lib.nb_get_body_contact_impulses.argtypes = [V, V, C.c_uint32, V, C.c_int, V]
        lib.nb_get_contact_pair_impulses.argtypes = [V, C.c_float, V, C.c_uint32, V, C.c_int, V]
        _lib = lib
    return _lib


class SpawnTables(C.Structure):
    _fields_ = [("filters", C.c_void_p), ("sensor_flags", C.c_void_p)]


class NudgeError(RuntimeError):
    pass


class Snapshot:
    """A device-resident snapshot of one Sim (nb_snapshot_*, include/nudge_b200.h): its handle, and the Sim's scene as of the last save.
    Sim.snapshot() makes one; Sim.snapshot(into=snap) saves into an existing one, Sim.restore(snap) goes back to it.  Freed by close(), when
    collected, or with its Sim."""

    def __init__(self, sim):
        self.sim = sim
        self.handle = C.c_void_p()
        self.scene = None
        sim._ck(sim.lib.nb_snapshot_create(sim.ctx, C.byref(self.handle)), "nb_snapshot_create")

    def close(self):
        if self.handle and self.sim.ctx:   # a closed Sim has freed its snapshots (nb_destroy)
            self.sim.lib.nb_snapshot_destroy(self.handle)
        self.handle = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


# nb_constraint_row (80 bytes)
ROW = np.dtype([("a", "<u4"), ("b", "<u4"), ("lin_a", "<f4", 3), ("ang_a", "<f4", 3), ("lin_b", "<f4", 3), ("ang_b", "<f4", 3),
                ("bias", "<f4"), ("lo", "<f4"), ("hi", "<f4"), ("impulse", "<f4"), ("softness", "<f4"), ("reserved", "<f4")])
assert ROW.itemsize == 80
JOINT = abi.JOINT
JOINT_BALL, JOINT_HINGE, JOINT_FIXED, JOINT_DISTANCE = 0, 1, 2, 3
JOINT_DRIVE = abi.JOINT_DRIVE
JOINT_LIMIT, JOINT_MOTOR, JOINT_BREAKABLE, JOINT_SLIDE, JOINT_CONE, JOINT_TWIST = 1, 2, 4, 16, 32, 64
JOINT_SPRING = abi.JOINT_SPRING


def nccl_unique_id():
    """128 bytes from ncclGetUniqueId (rank 0 calls it and broadcasts them)."""
    buf = (C.c_ubyte * 128)()
    r = load_library().nb_shard_unique_id(buf)
    if r != 0:
        raise NudgeError("nb_shard_unique_id failed (%d): NCCL not loadable" % r)
    return bytes(buf)


def shard_partition(pos, radius, gx, gz, margin, balance=0):
    """nb_shard_partition (C++ host code, runs without a GPU): owner[n] and the ghost list of every rank."""
    lib = load_library()
    pos = np.ascontiguousarray(pos, np.float32); radius = np.ascontiguousarray(radius, np.float32)
    n, world = len(radius), gx * gz
    owner = np.zeros(n, np.uint32); off = np.zeros(world + 1, np.uint32)
    cap = max(1024, n)
    while True:
        ids = np.zeros(cap, np.uint32)
        r = lib.nb_shard_partition(abi.ptr(pos), abi.ptr(radius), n, int(gx), int(gz), C.c_float(margin), int(balance), abi.ptr(owner), abi.ptr(off), abi.ptr(ids), cap)
        if r == 0:
            break
        if r != -2:
            raise NudgeError("nb_shard_partition failed (%d)" % r)
        cap = int(off[world]) + 16
    return owner, [ids[off[k]:off[k + 1]].copy() for k in range(world)]


def shard_build_plan(owner, ghost_lists, rank):
    """nb_shard_build_plan (C++ host code, runs without a GPU): the exchange plan of `rank` from a partition (owner[n], one 0-based ascending
    ghost id list per rank).  Returns a dict with the arrays nb_shard_plan takes plus owned_ids and max_export."""
    lib = load_library()
    owner = np.ascontiguousarray(owner, np.uint32)
    world = len(ghost_lists)
    off = np.zeros(world + 1, np.uint32)
    off[1:] = np.cumsum([len(g) for g in ghost_lists])
    ids = np.ascontiguousarray(np.concatenate([np.asarray(g, np.uint32) for g in ghost_lists]) if off[world] else np.zeros(1, np.uint32), np.uint32)
    sizes = (C.c_uint32 * 5)()
    r = lib.nb_shard_build_plan(abi.ptr(owner), len(owner), abi.ptr(off), abi.ptr(ids), world, int(rank), sizes, None, None, None, None, None, None, None)
    if r != 0:
        raise NudgeError("nb_shard_build_plan failed (%d)" % r)
    n_owned, n_export, n_ghost, n_sub, max_export = (int(x) for x in sizes)
    A = lambda k: np.zeros(max(int(k), 1), np.uint32)
    owned, exp, so, sr, ss, gl, gs = A(n_owned), A(n_export), A(n_export + 1), A(n_sub), A(n_sub), A(n_ghost), A(n_ghost)
    r = lib.nb_shard_build_plan(abi.ptr(owner), len(owner), abi.ptr(off), abi.ptr(ids), world, int(rank), sizes, abi.ptr(owned), abi.ptr(exp), abi.ptr(so), abi.ptr(sr), abi.ptr(ss), abi.ptr(gl), abi.ptr(gs))
    if r != 0:
        raise NudgeError("nb_shard_build_plan failed (%d)" % r)
    return dict(owned_ids=owned[:n_owned], export_local=exp[:n_export], sub_off=so[:n_export + 1], sub_rank=sr[:n_sub], sub_slot=ss[:n_sub],
                ghost_local=gl[:n_ghost], ghost_src=gs[:n_ghost], max_export=max_export)


def shard_local_scene(owned_ids, ghost_ids, n_bodies_global, box_body, sphere_body):
    """nb_shard_local_scene (C++ host code): (box_sel, box_local_body, sphere_sel, sphere_local_body) for the local scene
    [world body, owned_ids + 1 ..., ghost_ids + 1 ...] (ids 0-based as in shard_partition)."""
    lib = load_library()
    o = np.ascontiguousarray(owned_ids, np.uint32); g = np.ascontiguousarray(ghost_ids, np.uint32)
    bb = np.ascontiguousarray(box_body, np.uint32); sb = np.ascontiguousarray(sphere_body, np.uint32)
    P = lambda a: abi.ptr(a) if len(a) else None
    sizes = (C.c_uint32 * 2)()
    r = lib.nb_shard_local_scene(P(o), len(o), P(g), len(g), int(n_bodies_global), P(bb), len(bb), P(sb), len(sb), sizes, None, None, None, None)
    if r != 0:
        raise NudgeError("nb_shard_local_scene failed (%d)" % r)
    kb, ks = int(sizes[0]), int(sizes[1])
    A = lambda k: np.zeros(max(k, 1), np.uint32)
    bsel, bloc, ssel, sloc = A(kb), A(kb), A(ks), A(ks)
    r = lib.nb_shard_local_scene(P(o), len(o), P(g), len(g), int(n_bodies_global), P(bb), len(bb), P(sb), len(sb), sizes, abi.ptr(bsel), abi.ptr(bloc), abi.ptr(ssel), abi.ptr(sloc))
    if r != 0:
        raise NudgeError("nb_shard_local_scene failed (%d)" % r)
    return bsel[:kb], bloc[:kb], ssel[:ks], sloc[:ks]


class Sim(abi.HostState):
    """Device-resident simulation mirroring the reference's call sequence (example/main.cpp:274-328).

    Host arrays (self.transforms, self.momentum, ...) are the caller-owned copies; `upload()` / `download_bodies()`
    move them across.  `stream` is a raw cudaStream_t (0 = default stream)."""

    def __init__(self, scene, contact_capacity=None, pair_capacity=None, device=0, stream=0, debug=False, max_bodies=None, max_boxes=None, max_spheres=None):
        """max_* reserve room for scenes loaded later with reload() (a sharded scene changes size when it is re-partitioned)."""
        mb, mx, ms = max(scene.n_bodies, max_bodies or 0), max(scene.n_boxes, max_boxes or 0), max(scene.n_spheres, max_spheres or 0)
        super().__init__(scene, contact_capacity or max(1024, 24 * mb))
        self.lib = load_library()
        self.stream = C.c_void_p(stream)
        self.event_capacity = 0
        cfg = Config(mb, mx, ms, max(1, len(scene.connections)),
                     pair_capacity or max(4096, 16 * (mx + ms)), self.cap, device)
        self.ctx = C.c_void_p()
        r = self.lib.nb_create(C.byref(cfg), C.byref(self.ctx))
        if r != 0:
            msg = self.lib.nb_last_error(self.ctx).decode() if self.ctx else "nb_create failed"
            raise NudgeError("nb_create: %s (%d)" % (msg, r))
        if debug:
            self._ck(self.lib.nb_debug_enable(self.ctx, 1), "nb_debug_enable")
        self.upload()

    def close(self):
        if getattr(self, "shard", None):
            self.lib.nb_shard_destroy(self.shard)
            self.shard = None
        if getattr(self, "ctx", None):
            self.lib.nb_destroy(self.ctx)
            self.ctx = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _ck(self, r, what):
        if r != 0:
            raise NudgeError("%s: %s (%d)" % (what, self.lib.nb_last_error(self.ctx).decode(), r))

    def reload(self, scene):
        """Replaces the scene (bodies and colliders) inside the same device context; the contact cache in HBM is kept (it is keyed by collider tags)."""
        cap = self.cap
        abi.HostState.__init__(self, scene, cap)
        self._ck(self.lib.nb_upload_bodies(self.ctx, C.byref(self.bodies), self.stream), "nb_upload_bodies")
        self._ck(self.lib.nb_upload_colliders(self.ctx, C.byref(self.colliders), self.stream), "nb_upload_colliders")
        self._ck(self.lib.nb_upload_connections(self.ctx, C.byref(self.conn), self.stream), "nb_upload_connections")
        self._upload_scene_filters()

    def pack_momentum(self, dev_indices_ptr, n, dev_out_ptr):
        self._ck(self.lib.nb_pack_momentum(self.ctx, C.c_void_p(dev_indices_ptr), int(n), C.c_void_p(dev_out_ptr), self.stream), "nb_pack_momentum")

    def unpack_momentum(self, dev_indices_ptr, dev_sources_ptr, n, dev_in_ptr):
        self._ck(self.lib.nb_unpack_momentum(self.ctx, C.c_void_p(dev_indices_ptr), C.c_void_p(dev_sources_ptr), int(n), C.c_void_p(dev_in_ptr), self.stream), "nb_unpack_momentum")

    # ---- one scene sharded across GPUs: the C++ host behind nb_shard_* (include/nudge_b200.h) ----
    TRANSPORT = {"nccl": 0, "peer": 1}

    def shard_create(self, rank, world, nccl_id, ghost_capacity, export_capacity):
        self.shard = C.c_void_p()
        idbuf = (C.c_ubyte * 128).from_buffer_copy(nccl_id) if nccl_id is not None else None
        self._ck(self.lib.nb_shard_create(self.ctx, int(rank), int(world), idbuf, int(ghost_capacity), int(export_capacity), C.byref(self.shard)), "nb_shard_create")

    def shard_ipc_handle(self):
        h = (C.c_ubyte * 64)()
        self._ck(self.lib.nb_shard_ipc_handle(self.shard, h), "nb_shard_ipc_handle")
        return bytes(h)

    def shard_open_peer(self, peer, handle):
        self._ck(self.lib.nb_shard_open_peer(self.shard, int(peer), (C.c_ubyte * 64).from_buffer_copy(handle)), "nb_shard_open_peer")

    def shard_plan(self, export_local, sub_off, sub_rank, sub_slot, ghost_local, ghost_src, max_export):
        arrs = [np.ascontiguousarray(x, np.uint32) for x in (export_local, sub_off, sub_rank, sub_slot, ghost_local, ghost_src)]
        e, so, sr, ss, gl, gs = arrs
        self._ck(self.lib.nb_shard_plan(self.shard, abi.ptr(e), len(e), abi.ptr(so), abi.ptr(sr), abi.ptr(ss), abi.ptr(gl), abi.ptr(gs), len(gl), int(max_export), self.stream), "nb_shard_plan")

    def shard_exchange(self, transport):
        self._ck(self.lib.nb_shard_exchange(self.shard, self.TRANSPORT[transport], self.stream), "nb_shard_exchange")

    def shard_step(self, transport):
        s = self.scene
        self._ck(self.lib.nb_shard_step(self.shard, float(s.time_step), int(s.iterations), float(s.gravity), float(s.damping), self.TRANSPORT[transport], self.stream), "nb_shard_step")

    def shard_no_exchange(self, on):
        self._ck(self.lib.nb_shard_debug_no_exchange(self.shard, 1 if on else 0), "nb_shard_debug_no_exchange")

    def shard_graph_active(self):
        return bool(self.lib.nb_shard_graph_active(self.shard))

    # ---- host <-> HBM ----
    def upload(self):
        self._ck(self.lib.nb_upload_bodies(self.ctx, C.byref(self.bodies), self.stream), "nb_upload_bodies")
        self._ck(self.lib.nb_upload_colliders(self.ctx, C.byref(self.colliders), self.stream), "nb_upload_colliders")
        self._ck(self.lib.nb_upload_connections(self.ctx, C.byref(self.conn), self.stream), "nb_upload_connections")
        self._ck(self.lib.nb_upload_cache(self.ctx, C.byref(self.cache), self.stream), "nb_upload_cache")
        self._upload_scene_filters()

    def _upload_scene_filters(self):
        s = self.scene
        if getattr(s, "collision_filters", None) is not None or getattr(s, "filter_flags", 0):
            self.upload_collision_filters(s.collision_filters, s.filter_flags)
        if getattr(s, "sensors", None) is not None:
            self.upload_sensors(s.sensors)
        if getattr(s, "kinematic", None) is not None:
            self.upload_kinematic_bodies(s.kinematic)
        if getattr(s, "body_forces", None) is not None:
            rows = s.body_forces
            self.clear_body_forces()   # every body not listed gets the default entry
            self.set_body_forces(rows)

    def upload_bodies(self):
        self._ck(self.lib.nb_upload_bodies(self.ctx, C.byref(self.bodies), self.stream), "nb_upload_bodies")

    def upload_cache(self):
        self._ck(self.lib.nb_upload_cache(self.ctx, C.byref(self.cache), self.stream), "nb_upload_cache")

    def download_bodies(self):
        self._ck(self.lib.nb_download_bodies(self.ctx, C.byref(self.bodies), self.stream), "nb_download_bodies")

    def download_contacts(self):
        self.contacts.capacity = self.cap
        self.active.capacity = self.scene.n_bodies
        self._ck(self.lib.nb_download_contacts(self.ctx, C.byref(self.contacts), C.byref(self.active), self.stream), "nb_download_contacts")

    def download_cache(self):
        self.cache.capacity = self.cap
        self._ck(self.lib.nb_download_cache(self.ctx, C.byref(self.cache), self.stream), "nb_download_cache")

    def counts(self):
        c = Counts()
        r = self.lib.nb_download_counts(self.ctx, C.byref(c), self.stream)
        if r != -4:   # NB_ERR_OVERFLOW still fills the struct: the caller reads c.overflow
            self._ck(r, "nb_download_counts")
        return c

    # ---- the seven calls + the user loop ----
    def collide(self):
        self._ck(self.lib.nb_collide(self.ctx, self.stream), "nb_collide")

    def apply_gravity_damping(self):
        s = self.scene
        self._ck(self.lib.nb_apply_gravity_damping(self.ctx, float(s.time_step), float(s.gravity), float(s.damping), self.stream), "nb_apply_gravity_damping")

    def read_cached_impulses(self):
        self._ck(self.lib.nb_read_cached_impulses(self.ctx, self.stream), "nb_read_cached_impulses")

    def setup_contact_constraints(self):
        self._ck(self.lib.nb_setup_contact_constraints(self.ctx, self.stream), "nb_setup_contact_constraints")

    def apply_impulses(self, sweeps=1):
        self._ck(self.lib.nb_apply_impulses(self.ctx, int(sweeps), self.stream), "nb_apply_impulses")

    def update_cached_impulses(self):
        self._ck(self.lib.nb_update_cached_impulses(self.ctx, self.stream), "nb_update_cached_impulses")

    def write_cached_impulses(self):
        self._ck(self.lib.nb_write_cached_impulses(self.ctx, self.stream), "nb_write_cached_impulses")

    def advance(self):
        self._ck(self.lib.nb_advance(self.ctx, float(self.scene.time_step), self.stream), "nb_advance")

    def step(self):
        s = self.scene
        self._ck(self.lib.nb_step(self.ctx, float(s.time_step), int(s.iterations), float(s.gravity), float(s.damping), self.stream), "nb_step")

    def step_staged(self):
        """The same sub-step through the seven stage calls (example/main.cpp:274-328)."""
        self.collide(); self.apply_gravity_damping(); self.read_cached_impulses(); self.setup_contact_constraints()
        self.apply_impulses(int(self.scene.iterations)); self.update_cached_impulses(); self.write_cached_impulses(); self.advance()

    def launch_count(self):
        return int(self.lib.nb_launch_count(self.ctx))

    # ---- user constraint rows (nb_constraint_row, include/nudge_b200.h) ----
    def upload_constraint_rows(self, rows):
        rows = np.ascontiguousarray(rows, ROW)
        self._ck(self.lib.nb_upload_constraint_rows(self.ctx, abi.ptr(rows) if len(rows) else None, len(rows), self.stream), "nb_upload_constraint_rows")

    def download_constraint_rows(self, n):
        rows = np.zeros(n, ROW)
        self._ck(self.lib.nb_download_constraint_rows(self.ctx, abi.ptr(rows) if n else None, n, self.stream), "nb_download_constraint_rows")
        return rows

    # ---- joints (nb_joint, include/nudge_b200.h): rows rebuilt from the transforms on the device every step ----
    def upload_joints(self, joints):
        """Replaces the joint set with `joints` (JOINT rows; none removes it).  Asynchronous; the array may be reused on return."""
        j = np.ascontiguousarray(np.asarray(joints if joints is not None else [], JOINT).reshape(-1))
        self._ck(self.lib.nb_upload_joints(self.ctx, abi.ptr(j) if len(j) else None, len(j), self.stream), "nb_upload_joints")

    def download_joints(self):
        """The joints in upload order, impulse = the current accumulated impulses of each joint's rows."""
        n = C.c_uint32(0)
        self.lib.nb_download_joints(self.ctx, None, 0, C.byref(n), self.stream)   # the count (NB_ERR_CAPACITY unless there are none)
        out = np.zeros(n.value, JOINT)
        self._ck(self.lib.nb_download_joints(self.ctx, abi.ptr(out) if len(out) else None, len(out), C.byref(n), self.stream), "nb_download_joints")
        return out

    def upload_joint_drives(self, drives):
        """Replaces the joint drive set (limits, motors, sliders, swing cones, twist limits, break thresholds) with `drives` (JOINT_DRIVE rows; none removes it).  Asynchronous."""
        d = np.ascontiguousarray(np.asarray(drives if drives is not None else [], JOINT_DRIVE).reshape(-1))
        self._ck(self.lib.nb_upload_joint_drives(self.ctx, abi.ptr(d) if len(d) else None, len(d), self.stream), "nb_upload_joint_drives")

    def download_joint_drives(self):
        """The drives in joint order with their rows' current impulses, position and broken flag."""
        n = C.c_uint32(0)
        self.lib.nb_download_joint_drives(self.ctx, None, 0, C.byref(n), self.stream)   # the count (NB_ERR_CAPACITY unless there are none)
        out = np.zeros(n.value, JOINT_DRIVE)
        self._ck(self.lib.nb_download_joint_drives(self.ctx, abi.ptr(out) if len(out) else None, len(out), C.byref(n), self.stream), "nb_download_joint_drives")
        return out

    def upload_joint_springs(self, springs):
        """Replaces the joint spring set (position targets with stiffness and damping) with `springs` (JOINT_SPRING rows; none removes it).
        Asynchronous; the array may be reused on return."""
        d = np.ascontiguousarray(np.asarray(springs if springs is not None else [], JOINT_SPRING).reshape(-1))
        self._ck(self.lib.nb_upload_joint_springs(self.ctx, abi.ptr(d) if len(d) else None, len(d), self.stream), "nb_upload_joint_springs")

    def download_joint_springs(self):
        """The springs in joint order with their rows' current impulses and position."""
        n = C.c_uint32(0)
        self.lib.nb_download_joint_springs(self.ctx, None, 0, C.byref(n), self.stream)   # the count (NB_ERR_CAPACITY unless there are none)
        out = np.zeros(n.value, JOINT_SPRING)
        self._ck(self.lib.nb_download_joint_springs(self.ctx, abi.ptr(out) if len(out) else None, len(out), C.byref(n), self.stream), "nb_download_joint_springs")
        return out

    # ---- renderer read-back (example/main.cpp:224-268): one column-major 4x4 model matrix per collider, boxes first, then spheres ----
    def instance_matrices(self, out=None, device_ptr=None, capacity=0):
        """Host destination (default): returns an (n, 16) float32 array.  device_ptr: writes into that device buffer (e.g. a mapped
        graphics resource) asynchronously on the Sim's stream and returns the collider count."""
        n = C.c_uint32(0)
        if device_ptr is not None:
            self._ck(self.lib.nb_instance_matrices(self.ctx, C.c_void_p(device_ptr), capacity, 1, C.byref(n), self.stream), "nb_instance_matrices")
            return int(n.value)
        k = self.scene.n_colliders
        if out is None:
            out = np.zeros((k, 16), np.float32)
        self._ck(self.lib.nb_instance_matrices(self.ctx, abi.ptr(out), len(out), 0, C.byref(n), self.stream), "nb_instance_matrices")
        return out[:n.value]

    # ---- ray casts (nb_raycast, include/nudge_b200.h): the closest hit of every ray against the colliders as the transforms stand ----
    def raycast(self, rays, flags=0, device_ptrs=None, n=None):
        """rays: abi.RAY rows; returns their abi.RAY_HIT rows (collider = body = tag = RAY_NO_HIT for a miss).  flags: RAY_SENSORS also tests
        sensor colliders.  device_ptrs=(rays_ptr, hits_ptr) with n: device buffers of n rays and n hits instead; the call is then asynchronous on
        the Sim's stream (capturable after a first call) and returns None."""
        return self._sweep("raycast", "rays", abi.RAY, rays, flags, device_ptrs, n)

    # ---- shape casts (nb_shapecast, include/nudge_b200.h): where a moving sphere or oriented box first touches a collider ----
    def shapecast(self, casts, flags=0, device_ptrs=None, n=None):
        """casts: abi.SHAPE_CAST rows; returns their abi.RAY_HIT rows (collider = body = tag = RAY_NO_HIT for a miss).  flags:
        SHAPECAST_SENSORS also tests sensor colliders.  device_ptrs=(casts_ptr, hits_ptr) with n: device buffers of n casts and n hits
        instead; the call is then asynchronous on the Sim's stream (capturable after a first scene query) and returns None."""
        return self._sweep("shapecast", "casts", abi.SHAPE_CAST, casts, flags, device_ptrs, n)

    def _sweep(self, name, what, dtype, rows, flags, device_ptrs, n):
        """Sim.raycast and Sim.shapecast: nb_<name> on `what` (rows of dtype) into as many abi.RAY_HIT rows."""
        fn = getattr(self.lib, "nb_" + name)
        if device_ptrs is not None:
            if n is None:
                raise ValueError("Sim.%s with device_ptrs needs n, the number of %s (and hits) the two device buffers hold" % (name, what))
            self._ck(fn(self.ctx, C.c_void_p(device_ptrs[0]), int(n), C.c_void_p(device_ptrs[1]), int(flags), 1, self.stream), "nb_" + name)
            return None
        r = np.ascontiguousarray(np.asarray(rows, dtype).reshape(-1))
        out = np.zeros(len(r), abi.RAY_HIT)
        P = lambda a: abi.ptr(a) if len(a) else None
        self._ck(fn(self.ctx, P(r), len(r), P(out), int(flags), 0, self.stream), "nb_" + name)
        return out

    # ---- continuous collision (nb_upload_ccd_bodies, include/nudge_b200.h): fast bodies stop where their swept sphere first hits ----
    def upload_ccd_bodies(self, rows):
        """rows: abi.CCD_BODY rows (or anything np.asarray turns into them, e.g. tuples (body, radius, motion_threshold, category, mask)), or
        None / empty to remove the set.  Every step, each listed awake body whose translation is longer than its threshold casts its sphere
        along it on the device and stops at the first collider it would reach.  Asynchronous; the array may be reused on return."""
        r = np.ascontiguousarray(np.asarray(rows if rows is not None else [], abi.CCD_BODY).reshape(-1))
        self._ck(self.lib.nb_upload_ccd_bodies(self.ctx, abi.ptr(r) if len(r) else None, len(r), self.stream), "nb_upload_ccd_bodies")

    def download_ccd_bodies(self):
        """The set as abi.CCD_BODY rows, ascending by body (none without a set)."""
        n = C.c_uint32(0)
        self.lib.nb_download_ccd_bodies(self.ctx, None, 0, C.byref(n), self.stream)   # the count (NB_ERR_CAPACITY unless there is no set)
        out = np.zeros(n.value, abi.CCD_BODY)
        self._ck(self.lib.nb_download_ccd_bodies(self.ctx, abi.ptr(out) if len(out) else None, len(out), C.byref(n), self.stream), "nb_download_ccd_bodies")
        return out

    # ---- body states (nb_get_body_states, nb_set_body_states, include/nudge_b200.h): gather and scatter of chosen bodies' poses and velocities ----
    def get_body_states(self, bodies=None, device_ptrs=None, n=None):
        """The abi.BODY_STATE rows of `bodies` (None: bodies 0 .. B-1): position, rotation, velocity, angular velocity and idle counter as
        they stand on the device.  device_ptrs=(bodies_ptr or None, out_ptr) with n: device buffers of n indices (None: bodies 0 .. n-1)
        and n rows instead; the call is then asynchronous on the Sim's stream (capturable) and returns None, and an index at or beyond the
        body count gives a row with body = REMOVED_BODY and zeros."""
        if device_ptrs is not None:
            if n is None:
                raise ValueError("Sim.get_body_states with device_ptrs needs n, the number of rows the device buffers hold")
            idx, out = device_ptrs
            self._ck(self.lib.nb_get_body_states(self.ctx, C.c_void_p(idx) if idx else None, int(n), C.c_void_p(out), 1, self.stream), "nb_get_body_states")
            return None
        idx = None if bodies is None else np.ascontiguousarray(np.asarray(bodies, np.uint32).reshape(-1))
        k = self.scene.n_bodies if idx is None else len(idx)
        out = np.zeros(k, abi.BODY_STATE)
        self._ck(self.lib.nb_get_body_states(self.ctx, abi.ptr(idx) if idx is not None and k else None, k, abi.ptr(out) if k else None, 0, self.stream),
                 "nb_get_body_states")
        return out

    def set_body_states(self, states, fields, device_ptrs=None, n=None):
        """Writes abi.BODY_STATE rows on the device in list order: fields BODY_POSE sets position and rotation (and wakes what the moved
        bodies touched through the contact cache or a connection), BODY_VELOCITY velocity and angular velocity; every listed dynamic body
        gets idle counter 0.  Host rows are checked first (NudgeError on body 0, a body at or beyond the body count or a non-finite selected
        field) and the call returns 0.  device_ptrs=(states_ptr, skipped_ptr or None) with n: device buffers instead; invalid entries are
        skipped, their number written to the uint32 at skipped_ptr, and the call returns None (asynchronous, capturable).  The host mirrors
        (self.transforms, self.momentum, self.idle) are not updated; download_bodies() fetches the device's rows."""
        if device_ptrs is not None:
            if n is None:
                raise ValueError("Sim.set_body_states with device_ptrs needs n, the number of rows the device buffer holds")
            rows, skipped = device_ptrs
            self._ck(self.lib.nb_set_body_states(self.ctx, C.c_void_p(rows), int(n), int(fields), C.c_void_p(skipped) if skipped else None, 1, self.stream),
                     "nb_set_body_states")
            return None
        r = np.ascontiguousarray(np.asarray(states, abi.BODY_STATE).reshape(-1))
        skipped = C.c_uint32(0)
        self._ck(self.lib.nb_set_body_states(self.ctx, abi.ptr(r) if len(r) else None, len(r), int(fields), C.byref(skipped), 0, self.stream), "nb_set_body_states")
        return int(skipped.value)

    # ---- contact impulse reports (nb_get_body_contact_impulses, nb_get_contact_pair_impulses, include/nudge_b200.h) ----
    def get_body_contact_impulses(self, bodies=None, device_ptrs=None, n=None):
        """The abi.BODY_CONTACT_IMPULSE rows of `bodies` (None: bodies 0 .. B-1): the net contact impulse and angular impulse (about the
        body's position) each body received in the last solved step, and its contact sides.  Divide by the time step for a force.
        device_ptrs=(bodies_ptr or None, out_ptr) with n: device buffers of n indices (None: bodies 0 .. n-1) and n rows instead; the call
        is then asynchronous on the Sim's stream (capturable) and returns None, and an index at or beyond the body count gives a row with
        body = REMOVED_BODY and zeros.  NudgeError when no solved step is there to report on."""
        if device_ptrs is not None:
            if n is None:
                raise ValueError("Sim.get_body_contact_impulses with device_ptrs needs n, the number of rows the device buffers hold")
            idx, out = device_ptrs
            self._ck(self.lib.nb_get_body_contact_impulses(self.ctx, C.c_void_p(idx) if idx else None, int(n), C.c_void_p(out), 1, self.stream),
                     "nb_get_body_contact_impulses")
            return None
        idx = None if bodies is None else np.ascontiguousarray(np.asarray(bodies, np.uint32).reshape(-1))
        k = self.scene.n_bodies if idx is None else len(idx)
        out = np.zeros(k, abi.BODY_CONTACT_IMPULSE)
        self._ck(self.lib.nb_get_body_contact_impulses(self.ctx, abi.ptr(idx) if idx is not None and k else None, k, abi.ptr(out) if k else None, 0,
                                                       self.stream), "nb_get_body_contact_impulses")
        return out

    def get_contact_pair_impulses(self, min_normal_impulse=-np.inf, device_ptrs=None, capacity=None):
        """The abi.CONTACT_PAIR_IMPULSE rows of the last solved step's touching pairs whose normal impulse is at least min_normal_impulse
        (-inf: every pair), by ascending tags.  capacity: room for that many rows; with too few, raises NudgeError; without one, the count
        is asked for first.  device_ptrs=(out_ptr, count_ptr) with capacity: a device buffer of capacity rows and a device uint32 for the
        count instead; the call is then asynchronous on the Sim's stream (capturable) and returns None."""
        thr = float(min_normal_impulse)
        if device_ptrs is not None:
            if capacity is None:
                raise ValueError("Sim.get_contact_pair_impulses with device_ptrs needs capacity, the number of rows the device buffer holds")
            out, count = device_ptrs
            self._ck(self.lib.nb_get_contact_pair_impulses(self.ctx, thr, C.c_void_p(out), int(capacity), C.c_void_p(count), 1, self.stream),
                     "nb_get_contact_pair_impulses")
            return None
        count = C.c_uint32(0)
        if capacity is None:
            r = self.lib.nb_get_contact_pair_impulses(self.ctx, thr, None, 0, C.byref(count), 0, self.stream)
            if r != -2:   # NB_ERR_CAPACITY: count holds the number of rows
                self._ck(r, "nb_get_contact_pair_impulses")
            capacity = count.value
        out = np.zeros(max(int(capacity), 1), abi.CONTACT_PAIR_IMPULSE)
        self._ck(self.lib.nb_get_contact_pair_impulses(self.ctx, thr, abi.ptr(out) if capacity else None, int(capacity), C.byref(count), 0, self.stream),
                 "nb_get_contact_pair_impulses")
        return out[:count.value].copy()

    # ---- overlap queries (nb_overlap, include/nudge_b200.h): which colliders touch each sphere or oriented box ----
    def overlap(self, queries, flags=0, capacity=None, device_ptrs=None, n=None):
        """queries: abi.OVERLAP_QUERY rows; returns (offsets, hits): offsets[q] .. offsets[q + 1] indexes query q's abi.OVERLAP_HIT rows, by
        ascending collider.  flags: OVERLAP_SENSORS also tests sensor colliders.  capacity: room for that many hits; without one, a call
        that needs more is repeated once with room for the total.  With a capacity that is too small, raises NudgeError.
        device_ptrs=(queries_ptr, hits_ptr, offsets_ptr) with n and capacity: device buffers of n queries, capacity hits and n + 1 offsets
        instead; the call is then asynchronous on the Sim's stream (capturable once the scratch holds the capacity) and returns None."""
        if device_ptrs is not None:
            if n is None or capacity is None:
                raise ValueError("Sim.overlap with device_ptrs needs n (queries) and capacity (hits) of the device buffers")
            q, h, o = (C.c_void_p(p) for p in device_ptrs)
            self._ck(self.lib.nb_overlap(self.ctx, q, int(n), h, int(capacity), o, int(flags), 1, self.stream), "nb_overlap")
            return None
        qs = np.ascontiguousarray(np.asarray(queries, abi.OVERLAP_QUERY).reshape(-1))
        P = lambda a: abi.ptr(a) if len(a) else None
        cap = int(capacity) if capacity is not None else max(1024, 16 * len(qs))
        for retry in (capacity is None, False):
            offsets = np.zeros(len(qs) + 1, np.uint32)
            hits = np.zeros(cap, abi.OVERLAP_HIT)
            r = self.lib.nb_overlap(self.ctx, P(qs), len(qs), P(hits), cap, abi.ptr(offsets), int(flags), 0, self.stream)
            if r == -2 and retry:   # NB_ERR_CAPACITY: offsets[n] holds the total
                cap = int(offsets[-1])
                continue
            self._ck(r, "nb_overlap")
            return offsets, hits[:offsets[-1]]

    def upload_collision_filters(self, filters, flags=0):
        """filters: one scenes.FILTER row (category, mask) per collider, boxes first then spheres, or None / empty to remove the table.
        flags: FILTER_SKIP_CONNECTED also rejects pairs whose bodies are joined by a connection.  Colliders i and j collide iff
        category_i & mask_j and category_j & mask_i are both nonzero."""
        f = np.zeros(0, scenes.FILTER) if filters is None else np.ascontiguousarray(filters, scenes.FILTER)
        self._ck(self.lib.nb_upload_collision_filters(self.ctx, abi.ptr(f) if len(f) else None, len(f), int(flags), self.stream), "nb_upload_collision_filters")

    # ---- sensor colliders (nb_upload_sensors, include/nudge_b200.h): overlap without force ----
    def upload_sensors(self, flags, max_pairs=0):
        """flags: one uint8 per collider, boxes first then spheres (nonzero = sensor), or None / empty to remove the table.  max_pairs =
        candidate sensor pairs per collide (0: 256 per sensor collider, at least 1024).  The overlaps are sensor_overlaps(); with contact
        events enabled, SENSOR_BEGIN / SENSOR_END events follow the contact events of every step."""
        f = np.zeros(0, np.uint8) if flags is None else np.ascontiguousarray(flags, np.uint8)
        self._ck(self.lib.nb_upload_sensors(self.ctx, abi.ptr(f) if len(f) else None, len(f), int(max_pairs), self.stream), "nb_upload_sensors")

    def sensor_overlaps(self):
        """The overlaps of the last collide as a scenes.SENSOR_OVERLAP array, ascending by tags."""
        n = C.c_uint32(0)
        out = np.zeros(1, scenes.SENSOR_OVERLAP)
        r = self.lib.nb_download_sensor_overlaps(self.ctx, abi.ptr(out), 1, C.byref(n), self.stream)
        if r == -2:   # NB_ERR_CAPACITY: *count says how many are stored
            out = np.zeros(n.value, scenes.SENSOR_OVERLAP)
            r = self.lib.nb_download_sensor_overlaps(self.ctx, abi.ptr(out), len(out), C.byref(n), self.stream)
        self._ck(r, "nb_download_sensor_overlaps")
        return out[:n.value].copy()

    # ---- kinematic bodies (nb_upload_kinematic_bodies, include/nudge_b200.h): driven at a set velocity, never pushed back ----
    def upload_kinematic_bodies(self, rows):
        """rows: scenes.KINEMATIC rows (or anything np.asarray turns into them, e.g. tuples (body, velocity, angular_velocity, 0)), or
        None / empty to remove the set.  Replaces the set and writes each body's velocity and angular velocity into its momentum row on the
        device; call it every step with the same bodies and new velocities to drive them."""
        k = np.ascontiguousarray(np.asarray(rows if rows is not None else [], scenes.KINEMATIC).reshape(-1))
        self._ck(self.lib.nb_upload_kinematic_bodies(self.ctx, abi.ptr(k) if len(k) else None, len(k), self.stream), "nb_upload_kinematic_bodies")

    # ---- body impulses (nb_apply_body_impulses, nb_apply_radial_impulse, include/nudge_b200.h): hits, kicks, explosions, waking ----
    def apply_body_impulses(self, rows):
        """rows: scenes.BODY_IMPULSE rows (or anything np.asarray turns into them, e.g. tuples (body, offset, impulse, angular_impulse, (0, 0))),
        applied on the device in list order: velocity += mass_inverse * impulse, angular velocity += world inverse inertia * (offset x impulse +
        angular_impulse), and the body woken (idle counter 0).  An empty list does nothing."""
        r = np.ascontiguousarray(np.asarray(rows if rows is not None else [], scenes.BODY_IMPULSE).reshape(-1))
        self._ck(self.lib.nb_apply_body_impulses(self.ctx, abi.ptr(r) if len(r) else None, len(r), self.stream), "nb_apply_body_impulses")

    def apply_radial_impulse(self, center, radius, impulse):
        """An explosion (impulse > 0) or implosion (impulse < 0) on the device: every dynamic body whose position lies within `radius` of
        `center` is woken and pushed along the line from the center with an impulse falling linearly from `impulse` to 0 at the radius."""
        e = np.zeros(1, scenes.RADIAL_IMPULSE)
        e["center"] = center; e["radius"] = radius; e["impulse"] = impulse
        self._ck(self.lib.nb_apply_radial_impulse(self.ctx, abi.ptr(e), self.stream), "nb_apply_radial_impulse")

    # ---- per-body forces (nb_set_body_forces, include/nudge_b200.h): gravity scale, damping, constant force and torque inside the step ----
    def set_body_forces(self, rows):
        """rows: scenes.BODY_FORCE rows (or anything np.asarray turns into them), one per listed body; every other body keeps its entry.  The
        first call creates the table with the default entry for every body.  Each listed body is woken.  sim.scene.body_forces follows."""
        r = np.ascontiguousarray(np.asarray(rows if rows is not None else [], scenes.BODY_FORCE).reshape(-1))
        self._ck(self.lib.nb_set_body_forces(self.ctx, abi.ptr(r) if len(r) else None, len(r), self.stream), "nb_set_body_forces")
        old = self.scene.body_forces if self.scene.body_forces is not None else np.zeros(0, scenes.BODY_FORCE)
        merged = np.concatenate([old[~np.isin(old["body"], r["body"])], r])
        merged["reserved"] = 0
        self._own_scene().body_forces = merged[np.argsort(merged["body"], kind="stable")]

    def clear_body_forces(self):
        """Removes the table: the step is again the one without per-body forces."""
        self._ck(self.lib.nb_clear_body_forces(self.ctx, self.stream), "nb_clear_body_forces")
        if self.scene.body_forces is not None:
            self._own_scene().body_forces = None

    def _own_scene(self):
        """sim.scene, copied once so that edits of its tables do not reach the caller's Scene."""
        if self.scene is not getattr(self, "_owned_scene", None):
            self.scene = self._owned_scene = self.scene.copy()
        return self.scene

    def download_body_forces(self):
        """The device's entries as scenes.BODY_FORCE rows, one per body (body = the row index); default rows without a table."""
        n = C.c_uint32(0)
        out = np.zeros(max(self.scene.n_bodies, 1), scenes.BODY_FORCE)
        r = self.lib.nb_download_body_forces(self.ctx, abi.ptr(out), len(out), C.byref(n), self.stream)
        if r == -2:   # NB_ERR_CAPACITY: *count says how many bodies there are
            out = np.zeros(n.value, scenes.BODY_FORCE)
            r = self.lib.nb_download_body_forces(self.ctx, abi.ptr(out), len(out), C.byref(n), self.stream)
        self._ck(r, "nb_download_body_forces")
        return out[:n.value].copy()

    # ---- spawning and despawning (nb_add_bodies, nb_remove_bodies, include/nudge_b200.h): the scene changes shape on the device ----
    def add_bodies(self, fragment, filters=None, sensors=None):
        """Appends the bodies and colliders of `fragment` (a scenes.Scene, e.g. from scenes.fragment) on the device: its bodies become
        bodies B .., its boxes and spheres follow the existing ones.  The fragment's collider `body` fields count from its own first body.
        filters / sensors: the fragment colliders' entries (boxes, then spheres) for the context's filter / sensor table, required while that
        table exists.  sim.scene and the host mirrors follow the edit (transforms, momentum and idle counters are the host mirrors' values)."""
        s, fr = self.scene, fragment
        B = s.n_bodies
        new = s.copy()
        for k in ("transforms", "properties", "momentum", "idle"):
            setattr(new, k, np.concatenate([getattr(self, k), getattr(fr, k)]))
        bx, sx = fr.box_transforms.copy(), fr.sphere_transforms.copy()
        bx["body"] += np.uint32(B); sx["body"] += np.uint32(B)
        for k, v in (("box_tags", fr.box_tags), ("box_data", fr.box_data), ("box_transforms", bx), ("sphere_tags", fr.sphere_tags),
                     ("sphere_data", fr.sphere_data), ("sphere_transforms", sx)):
            setattr(new, k, np.concatenate([getattr(s, k), v]))
        f = sn = None
        if filters is not None:
            f = np.ascontiguousarray(filters, scenes.FILTER)
            if s.collision_filters is not None:
                new.collision_filters = np.concatenate([s.collision_filters[:s.n_boxes], f[:fr.n_boxes], s.collision_filters[s.n_boxes:], f[fr.n_boxes:]])
        if sensors is not None:
            sn = np.ascontiguousarray(sensors, np.uint8)
            if s.sensors is not None:
                new.sensors = np.concatenate([s.sensors[:s.n_boxes], sn[:fr.n_boxes], s.sensors[s.n_boxes:], sn[fr.n_boxes:]])
        parts = [np.ascontiguousarray(a) for a in (fr.transforms, fr.properties, fr.momentum, fr.idle, fr.box_tags, fr.box_data, bx, fr.sphere_tags, fr.sphere_data, sx)]
        P = lambda a: abi.ptr(a) if len(a) else None
        bodies = abi.BodyData(P(parts[0]), P(parts[1]), P(parts[2]), P(parts[3]), fr.n_bodies)
        cols = abi.ColliderData(abi.Shapes(P(parts[4]), P(parts[5]), P(parts[6]), fr.n_boxes), abi.Shapes(P(parts[7]), P(parts[8]), P(parts[9]), fr.n_spheres))
        t = SpawnTables(P(f) if f is not None else None, P(sn) if sn is not None else None)
        self._ck(self.lib.nb_add_bodies(self.ctx, C.byref(bodies), C.byref(cols), C.byref(t), self.stream), "nb_add_bodies")
        self._mirror(new)

    def remove_bodies(self, indices):
        """Removes the listed bodies (never body 0), their colliders, the connections, user rows and kinematic entries naming them, and
        compacts every index on the device (include/nudge_b200.h, nb_remove_bodies).  Bodies touching a removed one through the contact cache
        or a connection are woken.  sim.scene and the host mirrors follow the edit (transforms, momentum and idle counters are the host
        mirrors' values; download_bodies() fetches the device's)."""
        idx = np.ascontiguousarray(np.asarray(indices, np.uint32).reshape(-1))
        self._ck(self.lib.nb_remove_bodies(self.ctx, abi.ptr(idx) if len(idx) else None, len(idx), self.stream), "nb_remove_bodies")
        if not len(idx):
            return
        s = self.scene
        keep = np.ones(s.n_bodies, bool); keep[idx] = False
        new = s.copy()
        for k in ("transforms", "properties", "momentum", "idle"):
            setattr(new, k, getattr(self, k)[keep].copy())
        kc = keep[np.concatenate([s.box_transforms["body"], s.sphere_transforms["body"]]).astype(np.int64)]
        for k, v in self.download_colliders().items():
            setattr(new, k, v)
        new.connections = self.download_connections()
        if s.collision_filters is not None:
            new.collision_filters = s.collision_filters[kc].copy()
        if s.sensors is not None:
            new.sensors = s.sensors[kc].copy()
        if s.kinematic is not None:
            rank = (np.cumsum(keep) - 1).astype(np.uint32)
            k = s.kinematic[keep[s.kinematic["body"].astype(np.int64)]].copy()
            k["body"] = rank[k["body"].astype(np.int64)]
            new.kinematic = k if len(k) else None
        if s.body_forces is not None:
            rank = (np.cumsum(keep) - 1).astype(np.uint32)
            f = s.body_forces[keep[s.body_forces["body"].astype(np.int64)]].copy()
            f["body"] = rank[f["body"].astype(np.int64)]
            new.body_forces = f
        self._mirror(new)

    def _mirror(self, scene):
        """Host mirrors for the edited scene; the contact capacity is kept."""
        abi.HostState.__init__(self, scene, self.cap)

    def download_colliders(self):
        """The device's colliders as a dict of Scene fields: box_tags, box_data, box_transforms, sphere_tags, sphere_data, sphere_transforms."""
        A = abi.aligned_array
        nb, ns = max(self.scene.n_boxes, 1), max(self.scene.n_spheres, 1)
        while True:
            out = dict(box_tags=A(nb, np.uint32), box_data=A(nb, scenes.BOX), box_transforms=A(nb, scenes.TRANSFORM),
                       sphere_tags=A(ns, np.uint32), sphere_data=A(ns, scenes.SPHERE), sphere_transforms=A(ns, scenes.TRANSFORM))
            h = abi.ColliderData(abi.Shapes(abi.ptr(out["box_tags"]), abi.ptr(out["box_data"]), abi.ptr(out["box_transforms"]), nb),
                                 abi.Shapes(abi.ptr(out["sphere_tags"]), abi.ptr(out["sphere_data"]), abi.ptr(out["sphere_transforms"]), ns))
            r = self.lib.nb_download_colliders(self.ctx, C.byref(h), self.stream)
            if r != -2:   # NB_ERR_CAPACITY: the counts say how much room is needed
                break
            nb, ns = max(h.boxes.count, 1), max(h.spheres.count, 1)
        self._ck(r, "nb_download_colliders")
        kb, ks = h.boxes.count, h.spheres.count
        return {k: v[:kb if k.startswith("box") else ks].copy() for k, v in out.items()}

    def download_connections(self):
        """The device's connections as a scenes.PAIR32 array."""
        n = max(len(self.scene.connections), 1)
        while True:
            out = abi.aligned_array(n, scenes.PAIR32)
            h = abi.Connections(abi.ptr(out), 0)
            r = self.lib.nb_download_connections(self.ctx, C.byref(h), n, self.stream)
            if r != -2:
                break
            n = max(h.count, 1)
        self._ck(r, "nb_download_connections")
        return out[:h.count].copy()

    # ---- contact events (nb_contact_event, include/nudge_b200.h): which collider pairs began or ended touching, computed on the device ----
    def enable_contact_events(self, capacity):
        """capacity = events held between two drains (0 disables); resets the stored events, the dropped count and the step counter."""
        self._ck(self.lib.nb_enable_contact_events(self.ctx, int(capacity)), "nb_enable_contact_events")
        self.event_capacity = int(capacity)

    def contact_events(self, capacity=None):
        """Drains the device buffer: (events as a scenes.CONTACT_EVENT array, number of events dropped since the last drain because the
        buffer was full).  The events are always the first of the sequence; a drain with dropped > 0 still empties the buffer."""
        cap = self.event_capacity if capacity is None else int(capacity)
        out = np.zeros(max(cap, 1), scenes.CONTACT_EVENT)
        n = C.c_uint32(0); dropped = C.c_uint32(0)
        r = self.lib.nb_download_contact_events(self.ctx, abi.ptr(out), cap, C.byref(n), C.byref(dropped), self.stream)
        if r != -4:   # NB_ERR_OVERFLOW fills the outputs: the caller reads `dropped`
            self._ck(r, "nb_download_contact_events")
        return out[:n.value].copy(), int(dropped.value)

    # ---- device-resident snapshots (nb_snapshot_save / nb_snapshot_restore, include/nudge_b200.h): rollback and re-simulation ----
    def snapshot(self, into=None):
        """Saves the whole between-steps state into a Snapshot in HBM (a new one, or `into`) and returns it: one kernel launch, no
        synchronisation.  The snapshot keeps a reference to sim.scene; the next edit of the scene copies it instead of changing it in place."""
        snap = into if into is not None else Snapshot(self)
        self._ck(self.lib.nb_snapshot_save(self.ctx, snap.handle, self.stream), "nb_snapshot_save")
        snap.scene = self.scene
        self._owned_scene = None   # shared with the snapshot from here on: _own_scene copies before the next edit
        return snap

    def restore(self, snap):
        """Makes the device state what it was at `snap`'s save, bit for bit.  sim.scene and the host mirrors become those of the save; the
        stage calls that read the last collide's outputs are refused until the next collide() or step()."""
        self._ck(self.lib.nb_snapshot_restore(self.ctx, snap.handle, self.stream), "nb_snapshot_restore")
        if snap.scene is not self.scene:
            self._mirror(snap.scene)
        self._owned_scene = None

    # ---- state files (nb_save_state / nb_load_state; tools/nb_replay steps them headless) ----
    def save_state(self, path):
        self._ck(self.lib.nb_save_state(self.ctx, os.fsencode(path), self.stream), "nb_save_state")

    def load_state(self, path):
        self._ck(self.lib.nb_load_state(self.ctx, os.fsencode(path), self.stream), "nb_load_state")

    # ---- solver mode (include/nudge_b200.h): "parity" = the reference's exact Gauss-Seidel order, "throughput" = mass-splitting Jacobi ----
    def set_solver_mode(self, mode):
        self._ck(self.lib.nb_set_solver_mode(self.ctx, {"parity": 0, "throughput": 1}[mode]), "nb_set_solver_mode")

    def solver_mode(self):
        return ["parity", "throughput"][int(self.lib.nb_get_solver_mode(self.ctx))]

    def timing_enable(self, on=True):
        self._ck(self.lib.nb_debug_timing_enable(self.ctx, 1 if on else 0), "nb_debug_timing_enable")

    def timing(self):
        """(launches, total milliseconds) of the dominant solver kernel since the last call (CUDA events inside the library)."""
        n = C.c_uint32(0); ms = C.c_float(0.0)
        self._ck(self.lib.nb_debug_timing(self.ctx, C.byref(n), C.byref(ms), self.stream), "nb_debug_timing")
        return int(n.value), float(ms.value)

    def lut_model_exact(self):
        return bool(self.lib.nb_lut_model_exact(self.ctx))

    # ---- parity-test introspection ----
    def debug(self, name, dtype):
        n = C.c_size_t(0)
        self._ck(self.lib.nb_debug_read(self.ctx, name.encode(), None, 0, C.byref(n), self.stream), "nb_debug_read")
        buf = np.zeros(max(n.value, 1), np.uint8)
        if n.value:
            self._ck(self.lib.nb_debug_read(self.ctx, name.encode(), abi.ptr(buf), n.value, C.byref(n), self.stream), "nb_debug_read")
        return buf[:n.value].view(dtype)

    def debug_scalar(self, name):
        v = np.zeros(1, np.uint32); n = C.c_size_t(0)
        self._ck(self.lib.nb_debug_read(self.ctx, name.encode(), abi.ptr(v), 4, C.byref(n), self.stream), "nb_debug_read")
        return int(v[0])

    def device_rcp(self, x, rsqrt=False):
        x = np.ascontiguousarray(x, np.float32); y = np.empty_like(x)
        for b in range(0, len(x), 1024):
            xs = np.ascontiguousarray(x[b:b + 1024]); ys = np.empty_like(xs)
            self._ck(self.lib.nb_debug_rcp(self.ctx, abi.ptr(xs), abi.ptr(ys), len(xs), 1 if rsqrt else 0), "nb_debug_rcp")
            y[b:b + 1024] = ys
        return y

    def device_sort(self, keys, vals=None, begin_bit=0, end_bit=64):
        keys = np.ascontiguousarray(keys, np.uint64).copy()
        v = np.ascontiguousarray(vals, np.uint32).copy() if vals is not None else None
        self._ck(self.lib.nb_debug_sort(self.ctx, abi.ptr(keys), abi.ptr(v) if v is not None else None, len(keys), begin_bit, end_bit), "nb_debug_sort")
        return keys, v

    def device_scan(self, data):
        d = np.ascontiguousarray(data, np.uint32).copy(); total = np.zeros(1, np.uint32)
        self._ck(self.lib.nb_debug_scan(self.ctx, abi.ptr(d), len(d), abi.ptr(total)), "nb_debug_scan")
        return d, int(total[0])

    def pairs_view(self):
        kbits = self.debug_scalar("kbits")
        keys = self.debug("pair_keys", np.uint64)
        return dict(lo=(keys & np.uint64((1 << kbits) - 1)).astype(np.uint32), hi=(keys >> np.uint64(kbits)).astype(np.uint32), order=self.debug("order", np.uint32))

    def impulses_view(self):
        return dict(sorted=self.debug("sorted", np.uint32), data=self.debug("impulses", scenes.IMPULSE),
                    culled_tags=self.debug("culled_tags", np.uint64), culled_features=self.debug("culled_features", np.uint32),
                    culled_data=self.debug("culled_data", scenes.IMPULSE))

    def constraints_view(self):
        """Rows and states per occupied slot (slot = batch*8 + lane, the reference's ContactConstraintV lane), keyed by contact index."""
        stride = self.debug_scalar("row_stride")
        slot_contact = self.debug("row_contact", np.uint32)
        used = np.nonzero(slot_contact != 0xffffffff)[0]
        planes = self.debug("row_planes", np.float32).reshape(39, stride)[:, used]
        states = self.debug("row_states", np.float32).reshape(3, stride)[:, used]
        sorted_c = self.debug("sorted", np.uint32)
        n = len(sorted_c)
        batch = np.zeros(n, np.uint32); batch[sorted_c] = self.debug("batch_of", np.uint32)
        slot = np.zeros(n, np.uint32); slot[sorted_c] = self.debug("slot_idx", np.uint32)
        return dict(contact=slot_contact[used], a=self.debug("row_a", np.uint32)[used], b=self.debug("row_b", np.uint32)[used], rows=planes.T.copy(), states=states.T.copy(),
                    batch_of_contact=batch, slot_of_contact=slot, slots=used.astype(np.uint32))
