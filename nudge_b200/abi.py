"""ctypes mirrors of the widened (32-bit index) SoA structs declared in include/nudge_b200.h.

Field-for-field these are nudge.h:29-129 with index widths changed (SURVEY.md §0.3):
contact tag uint64 = feature | A<<32 | B<<48  becomes  tags[i] = A | B<<32 plus features[i].
`HostState` owns 64-byte aligned numpy arrays for one scene in this layout (what example/main.cpp:360-388
allocates for the reference) and exposes the struct views that are passed across the C ABI."""
import ctypes as C
import numpy as np
from . import scenes as S


class ContactData(C.Structure):
    _fields_ = [("data", C.c_void_p), ("bodies", C.c_void_p), ("tags", C.c_void_p), ("features", C.c_void_p),
                ("capacity", C.c_uint32), ("count", C.c_uint32), ("sleeping_pairs", C.c_void_p), ("sleeping_count", C.c_uint32)]


class Shapes(C.Structure):
    _fields_ = [("tags", C.c_void_p), ("data", C.c_void_p), ("transforms", C.c_void_p), ("count", C.c_uint32)]


class ColliderData(C.Structure):
    _fields_ = [("boxes", Shapes), ("spheres", Shapes)]


class BodyData(C.Structure):
    _fields_ = [("transforms", C.c_void_p), ("properties", C.c_void_p), ("momentum", C.c_void_p), ("idle_counters", C.c_void_p), ("count", C.c_uint32)]


class Connections(C.Structure):
    _fields_ = [("data", C.c_void_p), ("count", C.c_uint32)]


class ContactCache(C.Structure):
    _fields_ = [("tags", C.c_void_p), ("features", C.c_void_p), ("data", C.c_void_p), ("capacity", C.c_uint32), ("count", C.c_uint32)]


class ActiveBodies(C.Structure):
    _fields_ = [("indices", C.c_void_p), ("capacity", C.c_uint32), ("count", C.c_uint32)]


# nb_joint (112 bytes)
JOINT = np.dtype([("type", "<u4"), ("a", "<u4"), ("b", "<u4"), ("anchor_a", "<f4", 3), ("anchor_b", "<f4", 3), ("axis_a", "<f4", 3), ("axis_b", "<f4", 3),
                  ("rel_rotation", "<f4", 4), ("length", "<f4"), ("beta", "<f4"), ("softness", "<f4"), ("impulse", "<f4", 6)])
assert JOINT.itemsize == 112

# nb_joint_drive (56 bytes); flags: NB_JOINT_LIMIT = 1, NB_JOINT_MOTOR = 2, NB_JOINT_BREAKABLE = 4, NB_JOINT_SLIDE = 16, NB_JOINT_CONE = 32,
# NB_JOINT_TWIST = 64
JOINT_DRIVE = np.dtype([("joint", "<u4"), ("flags", "<u4"), ("lower", "<f4"), ("upper", "<f4"), ("motor_speed", "<f4"), ("max_motor_torque", "<f4"),
                        ("break_force", "<f4"), ("break_torque", "<f4"), ("impulse", "<f4", 3), ("position", "<f4"), ("broken", "<u4"), ("cone", "<f4")])
assert JOINT_DRIVE.itemsize == 56

# nb_joint_spring (56 bytes)
JOINT_SPRING = np.dtype([("joint", "<u4"), ("reserved", "<u4"), ("target", "<f4", 4), ("target_velocity", "<f4"), ("stiffness", "<f4"), ("damping", "<f4"),
                         ("max_force", "<f4"), ("impulse", "<f4", 3), ("position", "<f4")])
assert JOINT_SPRING.itemsize == 56

# nb_ray, nb_ray_hit (48 bytes each)
RAY = np.dtype([("origin", "<f4", 3), ("max_t", "<f4"), ("direction", "<f4", 3), ("mask", "<u4"), ("ignore_body", "<u4"), ("reserved", "<u4", 3)])
RAY_HIT = np.dtype([("position", "<f4", 3), ("t", "<f4"), ("normal", "<f4", 3), ("collider", "<u4"), ("body", "<u4"), ("tag", "<u4"), ("reserved", "<u4", 2)])
assert RAY.itemsize == 48 and RAY_HIT.itemsize == 48
RAY_SENSORS = 1
RAY_NO_HIT = 0xffffffff

# nb_overlap_query (64 bytes), nb_overlap_hit (16 bytes)
OVERLAP_QUERY = np.dtype([("shape", "<u4"), ("center", "<f4", 3), ("rotation", "<f4", 4), ("half_extents", "<f4", 3), ("radius", "<f4"),
                          ("mask", "<u4"), ("ignore_body", "<u4"), ("reserved", "<u4", 2)])
OVERLAP_HIT = np.dtype([("query", "<u4"), ("collider", "<u4"), ("body", "<u4"), ("tag", "<u4")])
assert OVERLAP_QUERY.itemsize == 64 and OVERLAP_HIT.itemsize == 16
OVERLAP_SPHERE = 0
OVERLAP_BOX = 1
OVERLAP_SENSORS = 1

# nb_shape_cast (80 bytes): an overlap query's shape moved along direction up to max_t; its hits are abi.RAY_HIT rows
SHAPE_CAST = np.dtype([("shape", OVERLAP_QUERY), ("direction", "<f4", 3), ("max_t", "<f4")])
assert SHAPE_CAST.itemsize == 80
SHAPECAST_SENSORS = 1

# nb_ccd_body (16 bytes): a body whose translation each step is clamped at the first hit of its swept sphere (continuous collision)
CCD_BODY = np.dtype([("body", "<u4"), ("radius", "<f4"), ("motion_threshold", "<f4"), ("category", "<u2"), ("mask", "<u2")])
assert CCD_BODY.itemsize == 16

# nb_body_state (64 bytes): one row of nb_get_body_states / nb_set_body_states; fields: BODY_POSE = 1, BODY_VELOCITY = 2
BODY_STATE = np.dtype([("position", "<f4", 3), ("body", "<u4"), ("rotation", "<f4", 4), ("velocity", "<f4", 3), ("idle_counter", "<u4"),
                       ("angular_velocity", "<f4", 3), ("reserved", "<u4")])
assert BODY_STATE.itemsize == 64
BODY_POSE = 1
BODY_VELOCITY = 2


def ptr(a):
    return a.ctypes.data_as(C.c_void_p)


def aligned_array(n, dtype, align=64):
    dtype = np.dtype(dtype)
    raw = np.zeros(max(n, 1) * dtype.itemsize + align, np.uint8)
    off = (-raw.ctypes.data) % align
    return raw[off:off + max(n, 1) * dtype.itemsize].view(dtype)[:n]


class HostState:
    """Caller-owned host arrays for one scene in the widened layout."""

    def __init__(self, scene, contact_capacity=None):
        self.scene = scene
        nb = scene.n_bodies
        cap = contact_capacity or max(1024, nb * 24)
        self.cap = cap
        A = aligned_array
        self.transforms = A(nb, S.TRANSFORM); self.transforms[:] = scene.transforms
        self.properties = A(nb, S.PROPERTIES); self.properties[:] = scene.properties
        self.momentum = A(nb, S.MOMENTUM); self.momentum[:] = scene.momentum
        self.idle = A(nb, np.uint8); self.idle[:] = scene.idle
        self.box_tags = A(scene.n_boxes, np.uint32); self.box_tags[:] = scene.box_tags
        self.box_data = A(scene.n_boxes, S.BOX); self.box_data[:] = scene.box_data
        self.box_transforms = A(scene.n_boxes, S.TRANSFORM); self.box_transforms[:] = scene.box_transforms
        self.sphere_tags = A(scene.n_spheres, np.uint32); self.sphere_tags[:] = scene.sphere_tags
        self.sphere_data = A(scene.n_spheres, S.SPHERE); self.sphere_data[:] = scene.sphere_data
        self.sphere_transforms = A(scene.n_spheres, S.TRANSFORM); self.sphere_transforms[:] = scene.sphere_transforms
        self.connections = A(len(scene.connections), S.PAIR32); self.connections[:] = scene.connections
        self.contact_data = A(cap, S.CONTACT)
        self.contact_bodies = A(cap, S.PAIR32)
        self.contact_tags = A(cap, np.uint64)
        self.contact_features = A(cap, np.uint32)
        self.sleeping_pairs = A(cap, np.uint64)
        self.active_indices = A(nb, np.uint32)
        self.cache_tags = A(cap, np.uint64)
        self.cache_features = A(cap, np.uint32)
        self.cache_data = A(cap, S.IMPULSE)

        self.bodies = BodyData(ptr(self.transforms), ptr(self.properties), ptr(self.momentum), ptr(self.idle), nb)
        self.colliders = ColliderData(Shapes(ptr(self.box_tags), ptr(self.box_data), ptr(self.box_transforms), scene.n_boxes),
                                      Shapes(ptr(self.sphere_tags), ptr(self.sphere_data), ptr(self.sphere_transforms), scene.n_spheres))
        self.conn = Connections(ptr(self.connections), len(self.connections))
        self.contacts = ContactData(ptr(self.contact_data), ptr(self.contact_bodies), ptr(self.contact_tags), ptr(self.contact_features),
                                    cap, 0, ptr(self.sleeping_pairs), 0)
        self.active = ActiveBodies(ptr(self.active_indices), nb, 0)
        self.cache = ContactCache(ptr(self.cache_tags), ptr(self.cache_features), ptr(self.cache_data), cap, 0)

    def contacts_view(self):
        n = self.contacts.count
        return dict(count=n, data=self.contact_data[:n].copy(), bodies=self.contact_bodies[:n].copy(), tags=self.contact_tags[:n].copy(),
                    features=self.contact_features[:n].copy(), sleeping=self.sleeping_pairs[:self.contacts.sleeping_count].copy(),
                    active=self.active_indices[:self.active.count].copy())

    def cache_view(self):
        n = self.cache.count
        return dict(tags=self.cache_tags[:n].copy(), features=self.cache_features[:n].copy(), data=self.cache_data[:n].copy())

    def apply_gravity_damping(self):
        """The user loop of example/main.cpp:291-305, float32."""
        f = np.float32
        dt = f(self.scene.time_step)
        damping = f(f(1.0) - dt * f(self.scene.damping))
        idx = self.active_indices[:self.active.count].astype(np.int64)
        m = self.momentum
        m["velocity"][idx, 1] = m["velocity"][idx, 1] - f(f(self.scene.gravity) * dt)
        m["velocity"][idx] = m["velocity"][idx] * damping
        m["angular_velocity"][idx] = m["angular_velocity"][idx] * damping

    def export_state(self):
        s = self.scene.copy()
        s.transforms[:] = self.transforms; s.momentum[:] = self.momentum; s.idle[:] = self.idle
        return s


def wide_tag_to_ref(tags, features):
    """Widened (A | B<<32, feature) -> the reference's 64-bit tag feature | A<<32 | B<<48 (valid when tags < 65536)."""
    tags = np.asarray(tags, np.uint64)
    return np.asarray(features, np.uint64) | ((tags & np.uint64(0xffff)) << np.uint64(32)) | ((tags >> np.uint64(32)) << np.uint64(48))


def wide_pair_to_ref(pairs):
    pairs = np.asarray(pairs, np.uint64)
    return ((pairs & np.uint64(0xffff)) | ((pairs >> np.uint64(32)) << np.uint64(16))).astype(np.uint32)
