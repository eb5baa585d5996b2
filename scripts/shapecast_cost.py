"""What shape casts cost on the c2 pile (scenes.box_drop(65536), settled, nb_step graph replay on a created stream); DESIGN.md §8.16.

  (a) calls of 1, 1,024 and 65,536 casts with device pointers, dropped straight down onto the pile from above it: spheres of radius 0.5,
      and oriented boxes (random unit rotations, half extents 0.25 to 0.75); CUDA events, median of --reps calls, with the share that hits;
  (b) the host alternative for 1,024 sphere casts: nb_download_bodies, then oracle/shapecast_ref.py's numpy brute force, and whether it
      gives the same bytes as the device;
  (c) nb_step alone against nb_step plus one 1,024-sphere-cast call per step, alternating windows.
Prints one JSON line with the card's name, power limit and SM clock, read in the same run.  GPU only: without a CUDA device it refuses.
usage: python scripts/shapecast_cost.py [--presim 1500] [--reps 20] [--window 25] [--rounds 8]"""
import argparse, json, os, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
import numpy as np
from scripts.body_impulse_cost import card


def family(kind, n, xf, rng, abi):
    p = xf["position"][1:]
    lo, hi = p.min(axis=0), p.max(axis=0)
    c = np.zeros(n, abi.SHAPE_CAST)
    q = c["shape"]
    q["mask"] = 0xffffffff; q["ignore_body"] = abi.RAY_NO_HIT; q["rotation"][:, 3] = 1.0
    q["center"] = np.c_[rng.uniform(lo[0], hi[0], n), np.full(n, hi[1] + 5.0), rng.uniform(lo[2], hi[2], n)]
    if kind == "sphere":
        q["shape"] = abi.OVERLAP_SPHERE; q["radius"] = 0.5
    else:
        v = rng.normal(size=(n, 4)); v /= np.linalg.norm(v, axis=1, keepdims=True)
        q["shape"] = abi.OVERLAP_BOX; q["rotation"] = v; q["half_extents"] = rng.uniform(0.25, 0.75, (n, 3))
    c["direction"] = (0.0, -1.0, 0.0); c["max_t"] = 1e3
    return c


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--boxes", type=int, default=65536)
    ap.add_argument("--presim", type=int, default=1500)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--window", type=int, default=25)
    ap.add_argument("--rounds", type=int, default=8)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("shapecast_cost.py measures on a CUDA GPU (H100); there is none here and no CPU path")
    import nudge_b200
    from nudge_b200 import abi, scenes
    from oracle import shapecast_ref, raycast_ref
    st = torch.cuda.Stream()
    x = nudge_b200.Sim(scenes.box_drop(args.boxes, iterations=8, seed=2), stream=st.cuda_stream)
    for _ in range(args.presim):
        x.step()
    x.download_bodies()
    rng = np.random.default_rng(1)
    maxn = 65536
    d_c = torch.zeros(maxn * 80, dtype=torch.uint8, device="cuda")
    d_h = torch.zeros(maxn * 48, dtype=torch.uint8, device="cuda")
    ptrs = (d_c.data_ptr(), d_h.data_ptr())

    def timed(n):
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        ms = []
        for _ in range(args.reps):
            ev[0].record(st)
            x.shapecast(None, device_ptrs=ptrs, n=n)
            ev[1].record(st)
            ev[1].synchronize()
            ms.append(ev[0].elapsed_time(ev[1]))
        return float(np.median(ms))

    def load(c):
        d_c[:len(c) * 80].copy_(torch.from_numpy(c.view(np.uint8).copy()))
        torch.cuda.synchronize()

    res = dict(script="shapecast_cost", boxes=args.boxes, presim=args.presim, reps=args.reps, call_ms={}, hit_share={})
    for kind in ("sphere", "box"):
        for n in (1, 1024, maxn):
            load(family(kind, n, x.transforms, rng, abi)); timed(n)
            res["call_ms"]["%s_%d" % (kind, n)] = round(timed(n), 4)
            hits = d_h[:n * 48].cpu().numpy().view(abi.RAY_HIT)
            res["hit_share"]["%s_%d" % (kind, n)] = round(float((hits["collider"] != abi.RAY_NO_HIT).mean()), 3)
    res["fallbacks"] = x.debug_scalar("shapecast_fallbacks")
    c = family("sphere", 1024, x.transforms, rng, abi)
    t0 = time.perf_counter()
    x.download_bodies()
    want = shapecast_ref.cast(raycast_ref.Scene.of_sim(x), c)
    res["host_1024_sphere_ms"] = round(1e3 * (time.perf_counter() - t0), 1)
    res["host_equals_device"] = bool(x.shapecast(c).tobytes() == want.tobytes())
    load(c)
    rate = {"step": [], "step_plus_1024_casts": []}
    for _ in range(args.rounds):
        for k in rate:
            st.synchronize()
            t0 = time.perf_counter()
            for _ in range(args.window):
                x.step()
                if k != "step":
                    x.shapecast(None, device_ptrs=ptrs, n=1024)
            st.synchronize()
            rate[k].append(args.window / (time.perf_counter() - t0))
    res["steps_per_s"] = {k: [round(v, 1) for v in rate[k]] for k in rate}
    res["median_steps_per_s"] = {k: round(float(np.median(v)), 1) for k, v in rate.items()}
    res.update(card())
    print(json.dumps(res))
    x.close()


if __name__ == "__main__":
    main()
