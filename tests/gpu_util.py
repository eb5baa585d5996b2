"""Test infrastructure shared by the GPU tests: a side stream, the hash nb_replay prints, and the state-file layout of
nudge_b200/csrc/nb_state_api.cuh (the header builder is also used by the CPU tests of nb_state_info)."""
import struct
import numpy as np

# magic, version, bodies, boxes, spheres, connections, cache, solver_mode, reserved[8]
STATE_HEADER = struct.Struct("<8s15I")
# The sections of a state file in file order: name, element size in bytes, what counts the elements.  Each is padded with zeros to 16
# bytes.  The last three are present only when the header says so (filter reserved[1], sensor reserved[2], kinematic reserved[4]).
STATE_LAYOUT = (("transforms", 32, "bodies"), ("properties", 16, "bodies"), ("momentum", 32, "bodies"), ("idle", 1, "bodies"),
                ("box_tags", 4, "boxes"), ("box_data", 16, "boxes"), ("box_transforms", 32, "boxes"),
                ("sphere_tags", 4, "spheres"), ("sphere_data", 4, "spheres"), ("sphere_transforms", 32, "spheres"),
                ("connections", 8, "connections"), ("cache_tags", 8, "cache"), ("cache_features", 4, "cache"), ("cache_data", 16, "cache"),
                ("filter", 4, "colliders"), ("sensor", 1, "colliders"), ("kinematic", 4, "kinematic"))
OPTIONAL_SECTIONS = ("filter", "sensor", "kinematic")


def side_stream():
    """A new CUDA stream (nb_step captures its graph only on a stream of its own)."""
    import torch
    return torch.cuda.Stream().cuda_stream


def joint_rows(g):
    """The joints' own rows, then the drive rows per driven joint in table order: nb_debug_read's "joint_rows" and "joint_drive_rows"
    concatenated, the layout the restatements' row functions return."""
    import nudge_b200
    return np.concatenate([g.debug("joint_rows", nudge_b200.ROW), g.debug("joint_drive_rows", nudge_b200.ROW)])


def fnv1a(b):
    """64-bit FNV-1a, the hash tools/nb_replay prints of the transforms."""
    h = 1469598103934665603
    for x in b:
        h = ((h ^ x) * 1099511628211) & 0xffffffffffffffff
    return h


def state_header(version, reserved=(0,) * 8, counts=(1000, 600, 400, 7, 12345), solver_mode=0):
    """A state file header; counts = bodies, boxes, spheres, connections, cache entries."""
    return STATE_HEADER.pack(b"NBSTATE1", version, *counts, solver_mode, *reserved)


def _counts(bodies, boxes, spheres, connections, cache, kinematic=0):
    return dict(bodies=bodies, boxes=boxes, spheres=spheres, connections=connections, cache=cache, colliders=boxes + spheres, kinematic=kinematic)


def state_size(bodies, boxes, spheres, connections, cache, filters):
    """The length of a state file without sensors or kinematic bodies, with the filter table when `filters`."""
    n = _counts(bodies, boxes, spheres, connections, cache)
    return STATE_HEADER.size + sum((size * n[c] + 15) // 16 * 16 for name, size, c in STATE_LAYOUT
                                   if name not in OPTIONAL_SECTIONS or (filters and name == "filter"))


def state_file(counts, sections, version=1, reserved=(0,) * 8, solver_mode=0):
    """A whole state file rebuilt from the layout: the header, then every section of STATE_LAYOUT that `sections` (name -> bytes) holds,
    in the layout's order and padded.  counts = bodies, boxes, spheres, connections, cache entries."""
    n = _counts(*counts, kinematic=reserved[4])
    out = state_header(version, reserved, counts, solver_mode)
    for name, size, c in STATE_LAYOUT:
        if name in sections:
            b = bytes(sections[name])
            assert len(b) == size * n[c], name
            out += b + bytes(-len(b) % 16)
    return out
