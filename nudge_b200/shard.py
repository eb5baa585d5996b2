"""Python harness over the C++ multi-GPU host (include/nudge_b200.h nb_shard_*, nudge_b200/csrc/nb_shard*.cuh): one scene sharded
across GPUs (SURVEY.md §8e).  Used by tests and bench.py; everything that runs per step on the device path is in the library.

Every rank runs the complete exact-order pipeline (collide ... advance) on its OWNED bodies plus GHOST copies of the neighbours'
bodies near its cell.  A contact between bodies of two ranks exists on both; each rank applies its impulses to both bodies, and
after the warm start and after every sweep the ghost rows are overwritten with their owners' BodyMomentum rows
(nb_shard_exchange: one ncclAllGather, or the library's own peer-memory push/pull kernels).  Within a rank the Gauss-Seidel order is
exactly the reference's; across ranks the coupling is block-Jacobi, so world_size > 1 is not bit-identical to the single-GPU
trajectory (world_size 1 is; a rank's result is a deterministic function of the partition; tests/ pin both and bound the physical
difference).  Ghosts are integrated locally with their owner's momentum, so no transform exchange is needed inside a partition
epoch; `reshard()` re-partitions from the gathered global state.

Partition (nb_shard_partition, C++ host code): gx x gz cells of equal body count in the (x, z) plane; body i is a ghost of every
other cell within radius_i + max_radius + margin of its centre.  Transports: "nccl" / "peer" (device, through the C ABI) and "host"
(numpy + torch.distributed on host buffers: the CPU tests over gloo, and bench.py's parity check of the device transports)."""
import numpy as np
from . import scenes as S


def body_radius(g):
    """Bounding radius of every body about its origin (max over its colliders; box: |half extents|, sphere: radius, plus the collider offset)."""
    r = np.zeros(g.n_bodies, np.float32)
    if g.n_boxes:
        rb = np.linalg.norm(g.box_data["size"], axis=1) + np.linalg.norm(g.box_transforms["position"], axis=1)
        np.maximum.at(r, g.box_transforms["body"].astype(np.int64), rb.astype(np.float32))
    if g.n_spheres:
        rs = g.sphere_data["radius"] + np.linalg.norm(g.sphere_transforms["position"], axis=1)
        np.maximum.at(r, g.sphere_transforms["body"].astype(np.int64), rs.astype(np.float32))
    return r


def choose_grid(pos, world):
    """gx x gz = world minimising the total cut length for this scene's footprint (a thin wall gets world x 1, a square pile 4 x 2 ...)."""
    ex = float(pos[:, 0].max() - pos[:, 0].min()) + 1e-6; ez = float(pos[:, 2].max() - pos[:, 2].min()) + 1e-6
    best = None
    for gx in range(1, world + 1):
        if world % gx:
            continue
        gz = world // gx
        cost = (gx - 1) * ez + (gz - 1) * ex
        if best is None or cost < best[0]:
            best = (cost, gx, gz)
    return best[1], best[2]


def partition(g, world, margin=0.5, grid=None, balance=3):
    """Owned / ghost / export lists (global body ids, ascending) of every rank for scene `g` (body 0 = static world, on every rank)."""
    from . import shard_partition
    pos = g.transforms["position"][1:].astype(np.float32)
    rad = body_radius(g)[1:]
    gx, gz = grid if grid is not None else choose_grid(pos, world)
    assert gx * gz == world
    owner, ghost_idx = shard_partition(pos, rad, gx, gz, margin, balance)
    ids = np.arange(1, g.n_bodies, dtype=np.int64)
    owned = [ids[owner == r] for r in range(world)]
    ghosts = [ghost_idx[r].astype(np.int64) + 1 for r in range(world)]
    exported = np.zeros(g.n_bodies, bool)
    for r in range(world):
        exported[ghosts[r]] = True
    export = [owned[r][exported[owned[r]]] for r in range(world)]
    return dict(grid=(gx, gz), owner=owner.astype(np.int64), owned=owned, ghosts=ghosts, export=export)


def local_scene(g, owned, ghosts):
    """Local Scene of one rank: body 0 (static world) + owned + ghosts, and every collider (box or sphere) that sits on one of them,
    in the global collider order.  Colliders keep their GLOBAL tag, so every rank orders contacts the way the global scene would
    (box tags < sphere tags as in example/main.cpp:171)."""
    from . import shard_local_scene
    gids = np.concatenate([[0], owned, ghosts]).astype(np.int64)
    n = len(gids)
    # which colliders sit on those bodies, and the local index of their bodies: the C++ host (nb_shard_local_scene)
    kb, lb, ks, ls = shard_local_scene(np.asarray(owned, np.int64) - 1, np.asarray(ghosts, np.int64) - 1, g.n_bodies, g.box_transforms["body"], g.sphere_transforms["body"])
    s = S.Scene(n, len(kb), len(ks))
    s.name = g.name + "_shard"
    s.transforms[:] = g.transforms[gids]; s.properties[:] = g.properties[gids]; s.momentum[:] = g.momentum[gids]; s.idle[:] = g.idle[gids]
    s.box_data[:] = g.box_data[kb]; s.box_transforms[:] = g.box_transforms[kb]; s.box_tags[:] = g.box_tags[kb]
    s.box_transforms["body"] = lb
    s.sphere_data[:] = g.sphere_data[ks]; s.sphere_transforms[:] = g.sphere_transforms[ks]; s.sphere_tags[:] = g.sphere_tags[ks]
    s.sphere_transforms["body"] = ls
    for k in ("time_step", "iterations", "gravity", "damping", "filter_flags"):
        setattr(s, k, getattr(g, k))
    if g.collision_filters is not None:   # ghosts keep their global filter: every rank decides a cross-shard pair the same way
        s.collision_filters = np.concatenate([g.collision_filters[:g.n_boxes][kb], g.collision_filters[g.n_boxes:][ks]])
    if getattr(g, "sensors", None) is not None:   # selected like the filter rows (nb_shard_step itself refuses a context with sensors)
        s.sensors = np.concatenate([g.sensors[:g.n_boxes][kb], g.sensors[g.n_boxes:][ks]]).astype(np.uint8)
    return s, gids


def exchange_plan(part, rank, n_bodies):
    """The arrays nb_shard_plan takes for `rank` (local body order: [world body, owned..., ghosts...]; ghost j uses inbox slot j), built by
    the C++ host (nb_shard_build_plan); exchange_plan_numpy is the same rule restated in numpy (tests compare the two)."""
    from . import shard_build_plan
    p = shard_build_plan(part["owner"], [g - 1 for g in part["ghosts"]], rank)
    assert np.array_equal(p["owned_ids"].astype(np.int64) + 1, part["owned"][rank])
    del p["owned_ids"]
    return p


def exchange_plan_numpy(part, rank, n_bodies):
    """exchange_plan restated in numpy (test infrastructure for nb_shard_build_plan)."""
    world = len(part["owned"])
    exp, ghosts, owned = part["export"], part["ghosts"], part["owned"]
    max_export = max(1, max(len(e) for e in exp))
    pos_in_export = np.zeros(n_bodies, np.int64)
    for r in range(world):
        pos_in_export[exp[r]] = np.arange(len(exp[r]))
    owner_of = np.zeros(n_bodies, np.int64); owner_of[1:] = part["owner"]
    lid = np.zeros(n_bodies, np.int64)
    n_owned = len(owned[rank])
    lid[owned[rank]] = 1 + np.arange(n_owned)
    export_local = lid[exp[rank]].astype(np.uint32)
    ghost_local = (1 + n_owned + np.arange(len(ghosts[rank]))).astype(np.uint32)
    ghost_src = (owner_of[ghosts[rank]] * max_export + pos_in_export[ghosts[rank]]).astype(np.uint32)
    rows, ranks, slots = [], [], []
    for p in range(world):
        if p == rank:
            continue
        mine = owner_of[ghosts[p]] == rank
        rows.append(pos_in_export[ghosts[p][mine]]); ranks.append(np.full(int(mine.sum()), p, np.int64)); slots.append(np.nonzero(mine)[0])
    rows = np.concatenate(rows) if rows else np.zeros(0, np.int64)
    ranks = np.concatenate(ranks) if ranks else np.zeros(0, np.int64); slots = np.concatenate(slots) if slots else np.zeros(0, np.int64)
    order = np.lexsort((ranks, rows))
    sub_off = np.zeros(len(export_local) + 1, np.uint32)
    sub_off[1:] = np.cumsum(np.bincount(rows, minlength=len(export_local)))
    return dict(export_local=export_local, sub_off=sub_off, sub_rank=ranks[order].astype(np.uint32), sub_slot=slots[order].astype(np.uint32),
                ghost_local=ghost_local, ghost_src=ghost_src, max_export=max_export)


class ShardedSim:
    """One rank of a sharded simulation.  `make_sim(scene, max_bodies)` builds the per-rank simulator (nudge_b200.Sim on the GPU box; the
    CPU oracle in the gloo tests).  transport: "nccl" | "peer" (the C++ host, device resident) or "host" (numpy exchange through
    torch.distributed `group`, any simulator)."""

    def __init__(self, global_scene, rank, world, make_sim, margin=0.5, transport="host", group=None, grid=None, capacity_factor=1.6, nccl=True, balance=3):
        self.g = global_scene.copy()
        self.rank, self.world, self.margin, self.grid = rank, world, float(margin), grid
        self.make_sim = make_sim
        self.transport = transport
        self.group = group
        self.capacity_factor = capacity_factor
        self.balance = balance                 # re-cuts of the cells towards even owned + ghost counts (nb_shard_partition)
        self.nccl = nccl                       # False: create the C++ shard without an NCCL communicator (peer transport only)
        self.sim = None
        self.shard_ready = False
        self.exchange_rows = 0
        self._partition()

    # ---- partition bookkeeping ----
    def _partition(self):
        g = self.g
        self.part = partition(g, self.world, self.margin, self.grid, self.balance)
        owned, ghosts = self.part["owned"][self.rank], self.part["ghosts"][self.rank]
        scene, self.gids = local_scene(g, owned, ghosts)
        self.n_owned = len(owned)
        if self.sim is None:
            biggest = max(len(self.part["owned"][r]) + len(self.part["ghosts"][r]) for r in range(self.world))
            self.cap_bodies = int(self.capacity_factor * biggest) + 1024
            self.sim = self.make_sim(scene, max(self.cap_bodies, scene.n_bodies))
        else:
            self.sim.reload(scene)
        self.plan = exchange_plan(self.part, self.rank, g.n_bodies)
        self.max_export = self.plan["max_export"]
        self.export_local, self.ghost_local, self.ghost_source = self.plan["export_local"], self.plan["ghost_local"], self.plan["ghost_src"]
        self.exchange_rows = len(self.export_local)
        if self.transport in ("nccl", "peer", "device") and self.world > 1:
            self._setup_device()
        self._host_buffers = None

    def _setup_device(self):
        """Creates the C++ shard once (NCCL communicator + peer inboxes) and uploads the plan of the current partition."""
        import torch.distributed as dist
        import nudge_b200
        sim = self.sim
        if not self.shard_ready:
            ids = [nudge_b200.nccl_unique_id() if (self.rank == 0 and self.nccl) else None]
            if self.nccl:
                dist.broadcast_object_list(ids, src=0, group=self.group)
            sim.shard_create(self.rank, self.world, ids[0], self.cap_bodies, self.cap_bodies)
            handles = [None] * self.world
            dist.all_gather_object(handles, sim.shard_ipc_handle(), group=self.group)
            ok = True
            try:
                for p in range(self.world):
                    if p != self.rank:
                        sim.shard_open_peer(p, handles[p])
            except Exception as e:  # noqa: BLE001 - CUDA IPC can be unavailable (container settings, no peer access): use the collective
                ok = False; self.peer_error = repr(e)
            oks = [None] * self.world
            dist.all_gather_object(oks, ok, group=self.group)
            self.peer_ok = all(oks)
            if not self.peer_ok and self.transport == "peer":
                if not self.nccl:
                    raise RuntimeError("peer-memory inboxes could not be opened and the shard has no NCCL communicator: %s" % getattr(self, "peer_error", "a peer failed"))
                self.transport = "nccl"          # every rank takes the same decision: the flags were all-gathered
            self.shard_ready = True
        p = self.plan
        sim.shard_plan(p["export_local"], p["sub_off"], p["sub_rank"], p["sub_slot"], p["ghost_local"], p["ghost_src"], p["max_export"])

    # ---- ghost exchange ----
    def exchange(self, transport=None):
        if self.world == 1:
            return
        t = transport or self.transport
        if t in ("nccl", "peer"):
            self.sim.shard_exchange(t)
            return
        import torch, torch.distributed as dist   # host path: same plan, numpy gathers
        sim = self.sim
        if self._host_buffers is None:
            self._host_buffers = (torch.zeros((self.max_export, 8), dtype=torch.float32), torch.zeros((self.world * self.max_export, 8), dtype=torch.float32))
        t_export, t_gather = self._host_buffers
        sim.download_bodies()
        rows = sim.momentum.view(np.float32).reshape(-1, 8)
        t_export.numpy()[:len(self.export_local)] = rows[self.export_local.astype(np.int64)]
        parts = [t_gather[r * self.max_export:(r + 1) * self.max_export] for r in range(self.world)]
        dist.all_gather(parts, t_export, group=self.group)
        rows[self.ghost_local.astype(np.int64)] = t_gather.numpy()[self.ghost_source.astype(np.int64)]
        sim.upload_bodies()

    # ---- one simulation step (example/main.cpp:274-328) with the exchanges ----
    def step(self, transport=None):
        t = transport or self.transport
        if self.world > 1 and t in ("nccl", "peer"):
            self.sim.shard_step(t)          # the whole sharded sub-step inside the library (CUDA graph replay on a capturable stream)
            return
        sim = self.sim
        sim.collide(); sim.apply_gravity_damping(); sim.read_cached_impulses(); sim.setup_contact_constraints()
        self.exchange(t)
        for _ in range(int(self.g.iterations)):
            sim.apply_impulses()
            self.exchange(t)
        sim.update_cached_impulses(); sim.write_cached_impulses(); sim.advance()

    def launch_count(self):
        return self.sim.launch_count()

    # ---- gather the global state on every rank and re-partition ----
    def gather_global(self):
        sim = self.sim
        sim.download_bodies()
        g = self.g
        own = slice(1, 1 + self.n_owned)
        ids = self.gids[own]
        if self.world == 1:
            g.transforms[ids] = sim.transforms[own]; g.momentum[ids] = sim.momentum[own]; g.idle[ids] = sim.idle[own]
            return g
        import torch, torch.distributed as dist
        # every rank knows every rank's owned list (the partition is a deterministic function of the gathered state), so only the rows
        # travel: 32 B transform + 32 B momentum + 1 B idle counter per owned body, padded to the largest rank, one all_gather
        owned = self.part["owned"]
        cap = max(1, max(len(o) for o in owned))
        n = self.n_owned
        rec = np.zeros((cap, 65), np.uint8)
        rec[:n, 0:32] = sim.transforms[own].view(np.uint8).reshape(n, 32)
        rec[:n, 32:64] = sim.momentum[own].view(np.uint8).reshape(n, 32)
        rec[:n, 64] = sim.idle[own]
        out = torch.empty((self.world, cap, 65), dtype=torch.uint8)
        dist.all_gather([out[r] for r in range(self.world)], torch.from_numpy(rec), group=self.group)
        got = out.numpy()
        for r in range(self.world):
            i, k = owned[r], len(owned[r])
            g.transforms[i] = np.ascontiguousarray(got[r, :k, 0:32]).view(S.TRANSFORM).reshape(k)
            g.momentum[i] = np.ascontiguousarray(got[r, :k, 32:64]).view(S.MOMENTUM).reshape(k)
            g.idle[i] = got[r, :k, 64]
        return g

    def reshard(self):
        self.gather_global()
        self._partition()

    def local_counts(self):
        return dict(owned=self.n_owned, ghosts=len(self.gids) - 1 - self.n_owned, export=self.exchange_rows)
