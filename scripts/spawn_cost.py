"""What spawning and despawning cost on the c2 pile (scenes.box_drop(65536), settled, nb_step graph replay on a created stream); DESIGN.md §8.10.

1. Device time of one call: nb_remove_bodies of n random pile bodies, then nb_add_bodies of n boxes put back where they were (same size, tag,
   transform and momentum, so the pile stays the pile), for n = 1, 16, 1,024 and 16,384.  CUDA events around the work the call enqueues, and
   the host clock around the call and a stream synchronise.
2. Churn, in alternating windows of the same context: (a) steps alone; (b) every step removes the 16 oldest of a pool of falling projectiles
   and adds 16 new ones above the pile (nb_remove_bodies + nb_add_bodies); (c) the same edit as a host round trip: nb_download_bodies,
   nb_download_cache (for the wake set), the numpy edit, and nb_upload_bodies / nb_upload_colliders / nb_upload_connections (the c2 scene has
   no filter, sensor, kinematic or row tables to re-upload).
Prints one JSON line with the card's name, power limit and SM clock, read in the same run.  GPU only: without a CUDA device it refuses to run.
usage: python scripts/spawn_cost.py [--boxes 65536] [--presim 1500] [--window 200] [--rounds 3] [--reps 20] [--pool 480]"""
import argparse, ctypes, json, os, subprocess, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
import numpy as np


def card():
    out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout
    name, power, clock, max_clock = (x.strip() for x in out.strip().splitlines()[0].split(","))
    return dict(gpu=name, power_limit=power, sm_clock=clock, max_sm_clock=max_clock)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--boxes", type=int, default=65536)
    ap.add_argument("--presim", type=int, default=1500)
    ap.add_argument("--window", type=int, default=200, help="steps per timed churn window")
    ap.add_argument("--rounds", type=int, default=3, help="(a) / (b) / (c) window rounds")
    ap.add_argument("--reps", type=int, default=20, help="calls timed per n")
    ap.add_argument("--pool", type=int, default=480, help="projectiles in flight during churn")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("spawn_cost.py measures on a CUDA GPU (H100); there is none here and no CPU path")
    import nudge_b200
    from nudge_b200 import scenes, abi
    s = scenes.box_drop(args.boxes, iterations=8, seed=2)
    B0 = s.n_bodies
    room = max(16384, args.pool + 16)
    x = nudge_b200.Sim(s, stream=torch.cuda.Stream().cuda_stream, max_bodies=B0 + room, max_boxes=s.n_boxes + room)
    L, ctx, st = x.lib, x.ctx, x.stream
    ts = torch.cuda.ExternalStream(st.value)
    sync = lambda: x._ck(L.nb_stream_synchronize(ctx, st), "nb_stream_synchronize")
    for _ in range(args.presim):
        x.step()
    sync()
    rng = np.random.default_rng(1)
    state = dict(B=B0, tags=s.box_tags.copy(), sizes=s.box_data.copy())   # box k sits on body k (box 0 = the ground on body 0)

    def raw_add(xf, props, mom, idle, tags, boxes, box_xf):
        n = len(xf)
        arrs = [np.ascontiguousarray(a) for a in (xf, props, mom, idle, tags, boxes, box_xf)]
        bodies = abi.BodyData(*(abi.ptr(a) for a in arrs[:4]), n)
        cols = abi.ColliderData(abi.Shapes(abi.ptr(arrs[4]), abi.ptr(arrs[5]), abi.ptr(arrs[6]), n), abi.Shapes(None, None, None, 0))
        x._ck(L.nb_add_bodies(ctx, ctypes.byref(bodies), ctypes.byref(cols), None, st), "nb_add_bodies")

    def timed(fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        sync()
        t0 = time.perf_counter()
        e0.record(ts); fn(); e1.record(ts)
        sync()
        return 1e6 * (time.perf_counter() - t0), 1e3 * e0.elapsed_time(e1)

    # 1. per call: remove n pile bodies, put the same boxes back at the end
    per_call = {}
    for n in (1, 16, 1024, 16384):
        rm_h, rm_d, add_h, add_d = [], [], [], []
        for _ in range(args.reps):
            x.download_bodies()
            B = state["B"]
            idx = np.sort(rng.choice(np.arange(1, B), n, replace=False)).astype(np.uint32)
            ii = idx.astype(np.int64)
            back = (x.transforms[ii].copy(), x.properties[ii].copy(), x.momentum[ii].copy(), x.idle[ii].copy(), state["tags"][ii].copy(), state["sizes"][ii].copy())
            h, d = timed(lambda: x._ck(L.nb_remove_bodies(ctx, abi.ptr(idx), n, st), "nb_remove_bodies"))
            rm_h.append(h); rm_d.append(d)
            keep = np.ones(B, bool); keep[ii] = False
            B2 = B - n
            bx = np.zeros(n, scenes.TRANSFORM); bx["rotation"][:, 3] = 1; bx["body"] = B2 + np.arange(n, dtype=np.uint32)
            h, d = timed(lambda: raw_add(back[0], back[1], back[2], back[3], back[4], back[5], bx))
            add_h.append(h); add_d.append(d)
            state["tags"] = np.concatenate([state["tags"][keep], back[4]]); state["sizes"] = np.concatenate([state["sizes"][keep], back[5]])
            x.step()   # an edit is followed by a step before the next one
        med = lambda v: round(float(np.median(v)), 1)
        per_call["n_%d" % n] = dict(remove_host_us=med(rm_h), remove_device_us=med(rm_d), add_host_us=med(add_h), add_device_us=med(add_d))
    step_h = [timed(x.step) for _ in range(args.reps)]
    per_call["step"] = dict(host_us=round(float(np.median([a for a, _ in step_h])), 1), device_us=round(float(np.median([b for _, b in step_h])), 1))

    # 2. churn: a FIFO pool of projectiles after the pile bodies; every step the 16 oldest go and 16 new ones come
    x.download_bodies()
    B = state["B"]
    L_half = 15.0 * np.sqrt(args.boxes / 8191.0)
    tag0 = int(state["tags"].max()) + 1
    counter = [0]

    def projectiles(k):
        t = np.zeros(k, scenes.TRANSFORM); t["rotation"][:, 3] = 1
        t["position"] = np.stack([rng.uniform(-L_half, L_half, k), np.full(k, 40.0), rng.uniform(-L_half, L_half, k)], 1)
        size = np.full((k, 3), 0.25, np.float32)
        tags = (tag0 + (counter[0] + np.arange(k)) % (args.pool + 16)).astype(np.uint32)
        counter[0] += k
        m = np.zeros(k, scenes.MOMENTUM); m["velocity"][:, 1] = -5.0
        return t, scenes._box_props(size), m, np.zeros(k, np.uint8), tags, size

    def add_projectiles(k, base):
        t, p, m, idle, tags, size = projectiles(k)
        boxes = np.zeros(k, scenes.BOX); boxes["size"] = size
        bx = np.zeros(k, scenes.TRANSFORM); bx["rotation"][:, 3] = 1; bx["body"] = base + np.arange(k, dtype=np.uint32)
        return t, p, m, idle, tags, boxes, bx

    raw_add(*add_projectiles(args.pool, B))
    x.step(); sync()
    first = np.arange(B, B + 16, dtype=np.uint32)
    Bc = B + args.pool

    def device_churn():
        x._ck(L.nb_remove_bodies(ctx, abi.ptr(first), 16, st), "nb_remove_bodies")
        raw_add(*add_projectiles(16, Bc - 16))

    # the host round trip keeps full host copies of the scene, as an application without the calls must
    host = dict(props=None, tags=None, data=None, bxf=None)
    cache = abi.aligned_array(x.cap, np.uint64), abi.aligned_array(x.cap, np.uint32), abi.aligned_array(x.cap, scenes.IMPULSE)

    def host_churn():
        n = Bc
        xf, pr, mo, idl = (abi.aligned_array(n, d) for d in (scenes.TRANSFORM, scenes.PROPERTIES, scenes.MOMENTUM, np.uint8))
        bd = abi.BodyData(abi.ptr(xf), abi.ptr(pr), abi.ptr(mo), abi.ptr(idl), n)
        x._ck(L.nb_download_bodies(ctx, ctypes.byref(bd), st), "nb_download_bodies")
        cc = abi.ContactCache(abi.ptr(cache[0]), abi.ptr(cache[1]), abi.ptr(cache[2]), x.cap, 0)
        x._ck(L.nb_download_cache(ctx, ctypes.byref(cc), st), "nb_download_cache")
        keep = np.ones(n, bool); keep[B:B + 16] = False
        # wake set: cache keys pairing a kept collider's tag with a removed one (tags are unique here: box k on body k)
        tags = host["tags"]
        removed_tag = np.zeros(int(tags.max()) + 1, bool); removed_tag[tags[~keep]] = True
        body_of = np.zeros(len(removed_tag), np.int64); body_of[tags] = np.arange(n)
        k = cache[0][:cc.count]
        a, b = (k & np.uint64(0xffffffff)).astype(np.int64), (k >> np.uint64(32)).astype(np.int64)
        wake = np.zeros(n, bool)
        wake[body_of[a[removed_tag[b]]]] = True; wake[body_of[b[removed_tag[a]]]] = True
        wake[0] = False
        idl[wake] = 0
        t, p, m, i_, nt, boxes, bx = add_projectiles(16, Bc - 16)
        xf2 = np.concatenate([xf[keep], t]); pr2 = np.concatenate([host["props"][keep], p]); mo2 = np.concatenate([mo[keep], m]); id2 = np.concatenate([idl[keep], i_])
        host["props"] = pr2
        host["tags"] = np.concatenate([tags[keep], nt]); host["data"] = np.concatenate([host["data"][keep], boxes])
        host["bxf"] = np.concatenate([host["bxf"][keep], bx]); host["bxf"]["body"] = np.arange(n, dtype=np.uint32)
        arrs = [np.ascontiguousarray(v) for v in (xf2, pr2, mo2, id2, host["tags"], host["data"], host["bxf"])]
        bd2 = abi.BodyData(*(abi.ptr(v) for v in arrs[:4]), n)
        cd = abi.ColliderData(abi.Shapes(abi.ptr(arrs[4]), abi.ptr(arrs[5]), abi.ptr(arrs[6]), n), abi.Shapes(None, None, None, 0))
        x._ck(L.nb_upload_bodies(ctx, ctypes.byref(bd2), st), "nb_upload_bodies")
        x._ck(L.nb_upload_colliders(ctx, ctypes.byref(cd), st), "nb_upload_colliders")
        conn = abi.Connections(None, 0)
        x._ck(L.nb_upload_connections(ctx, ctypes.byref(conn), st), "nb_upload_connections")
        x._ck(L.nb_stream_synchronize(ctx, st), "sync")   # the host arrays must outlive the asynchronous upload

    def host_init():
        x.download_bodies()
        n = Bc
        host["props"] = np.zeros(n, scenes.PROPERTIES)
        # properties are never written on the device: rebuild them from the sizes the script tracks
        sizes = np.concatenate([state["sizes"]["size"], np.full((args.pool, 3), 0.25, np.float32)])
        host["props"][1:] = scenes._box_props(sizes[1:]); host["props"][0] = s.properties[0]
        cols = x.download_colliders()
        host["tags"], host["data"], host["bxf"] = cols["box_tags"], cols["box_data"], cols["box_transforms"]

    modes = dict(a=lambda: None, b=device_churn, c=host_churn)
    rate = {k: [] for k in modes}
    for _ in range(args.rounds):
        for kname, edit in modes.items():
            if kname == "c":
                host_init()
            sync()
            t0 = time.perf_counter()
            for i in range(args.window):
                edit()
                x.step()
            sync()
            rate[kname].append(args.window / (time.perf_counter() - t0))
    graph = x.debug_scalar("graph_active")
    med = {k: float(np.median(v)) for k, v in rate.items()}
    c = x.counts()
    res = dict(script="spawn_cost", boxes=args.boxes, presim=args.presim, window_steps=args.window, window_rounds=args.rounds, pool=args.pool,
               per_call=per_call, steps_per_s={k: [round(v, 1) for v in rate[k]] for k in rate}, median_steps_per_s={k: round(v, 1) for k, v in med.items()},
               churn_cost_per_step_us={k: round(1e6 * (1.0 / med[k] - 1.0 / med["a"]), 1) for k in "bc"},
               graph_active=graph, bodies=Bc, overflow=c.overflow, **card())
    print(json.dumps(res))
    x.close()


if __name__ == "__main__":
    main()
