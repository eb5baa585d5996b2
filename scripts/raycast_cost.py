"""What ray casts cost on the c2 pile (scenes.box_drop(65536), settled, nb_step graph replay on a created stream); DESIGN.md §8.14.

  (a) the build alone: one nb_raycast of a single degenerate ray (the build and a walk that tests nothing), CUDA events around the call;
  (b) calls of 1, 1,024, 65,536 and 1,048,576 rays with device pointers, in three families: down-rays onto the pile, lidar fans from inside
      the pile (origins at body centres), random long rays across the bounds; CUDA events, median of --reps calls;
  (c) the host alternative for 1,024 down-rays: nb_download_bodies and the colliders' world transforms, then the numpy brute force;
  (d) nb_step alone against nb_step plus one 65,536-ray call per step, alternating windows;
  (e) a scene with spheres whose grid is fine: 30,000 sub-metre boxes and balls (half extents and radii 0.15 to 0.35) dropped on the
      standard 400-half-extent ground, 65,536 and 1,048,576 rays of each family, with its grid level and the rays that fell back to testing
      every collider (nb_debug_read "ray_fallbacks"; every in-scene ray should walk the grid).
Prints one JSON line with the card's name, power limit and SM clock, read in the same run.  GPU only: without a CUDA device it refuses.
usage: python scripts/raycast_cost.py [--presim 1500] [--reps 20] [--window 25] [--rounds 8]"""
import argparse, json, os, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
import numpy as np
from scripts.body_impulse_cost import card


def family(kind, n, xf, rng, abi):
    p = xf["position"][1:]
    lo, hi = p.min(axis=0), p.max(axis=0)
    r = np.zeros(n, abi.RAY)
    r["mask"] = 0xffffffff; r["ignore_body"] = abi.RAY_NO_HIT
    if kind == "down":
        r["origin"] = np.c_[rng.uniform(lo[0], hi[0], n), np.full(n, hi[1] + 5.0), rng.uniform(lo[2], hi[2], n)]
        r["direction"] = (0.0, -1.0, 0.0); r["max_t"] = 1e4
    elif kind == "lidar":   # fans of 64 rays in a horizontal circle around body centres
        c = p[rng.integers(0, len(p), (n + 63) // 64)]
        a = np.arange(64) * (2 * np.pi / 64)
        r["origin"] = np.repeat(c, 64, axis=0)[:n]
        r["direction"] = np.tile(np.c_[np.cos(a), np.full(64, -0.05), np.sin(a)], ((n + 63) // 64, 1))[:n]; r["max_t"] = 100.0
    else:
        v = rng.normal(size=(n, 3)); v /= np.linalg.norm(v, axis=1, keepdims=True)
        r["origin"] = rng.uniform(lo, hi, (n, 3)); r["direction"] = v; r["max_t"] = 1e4
    return r


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
        sys.exit("raycast_cost.py measures on a CUDA GPU (H100); there is none here and no CPU path")
    import nudge_b200
    from nudge_b200 import abi, scenes
    from oracle import raycast_ref
    st = torch.cuda.Stream()
    x = nudge_b200.Sim(scenes.box_drop(args.boxes, iterations=8, seed=2), stream=st.cuda_stream)
    for _ in range(args.presim):
        x.step()
    x.download_bodies()
    rng = np.random.default_rng(1)
    maxn = 1 << 20
    d_rays = torch.zeros(maxn * 48, dtype=torch.uint8, device="cuda")
    d_hits = torch.zeros(maxn * 48, dtype=torch.uint8, device="cuda")
    ptrs = (d_rays.data_ptr(), d_hits.data_ptr())

    def timed(n):
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        ms = []
        for _ in range(args.reps):
            ev[0].record(st)
            x.raycast(None, device_ptrs=ptrs, n=n)
            ev[1].record(st)
            ev[1].synchronize()
            ms.append(ev[0].elapsed_time(ev[1]))
        return float(np.median(ms))

    def load(r):
        d_rays[:len(r) * 48].copy_(torch.from_numpy(r.view(np.uint8).copy()))
        torch.cuda.synchronize()

    bad = family("down", 1, x.transforms, rng, abi); bad["max_t"] = -1.0
    load(bad); timed(1)
    res = dict(script="raycast_cost", boxes=args.boxes, presim=args.presim, reps=args.reps, build_ms=round(timed(1), 4), call_ms={}, hit_fraction={})
    for kind in ("down", "lidar", "random"):
        for n in (1, 1024, 65536, maxn):
            r = family(kind, n, x.transforms, rng, abi)
            load(r); timed(n)
            res["call_ms"]["%s_%d" % (kind, n)] = round(timed(n), 4)
            if n == 65536:
                h = d_hits[:n * 48].cpu().numpy().view(abi.RAY_HIT)
                res["hit_fraction"][kind] = round(float((h["collider"] != abi.RAY_NO_HIT).mean()), 3)
    down = family("down", 1024, x.transforms, rng, abi)
    t0 = time.perf_counter()
    x.download_bodies()
    want = raycast_ref.cast(raycast_ref.Scene.of_sim(x), down)
    res["host_1024_down_ms"] = round(1e3 * (time.perf_counter() - t0), 1)
    res["host_equals_device"] = bool(want.tobytes() == x.raycast(down).tobytes())
    r = family("random", 65536, x.transforms, rng, abi)
    load(r)
    rate = {"step": [], "step_plus_65536_rays": []}
    for _ in range(args.rounds):
        for k in rate:
            st.synchronize()
            t0 = time.perf_counter()
            for _ in range(args.window):
                x.step()
                if k != "step":
                    x.raycast(None, device_ptrs=ptrs, n=65536)
            st.synchronize()
            rate[k].append(args.window / (time.perf_counter() - t0))
    res["steps_per_s"] = {k: [round(v, 1) for v in rate[k]] for k in rate}
    res["median_steps_per_s"] = {k: round(float(np.median(v)), 1) for k, v in rate.items()}
    x.close()
    rng2 = np.random.default_rng(3)
    nb = 15000
    pos = lambda k: np.stack([rng2.uniform(-25, 25, k), rng2.uniform(0, 30, k) - 9.0, rng2.uniform(-25, 25, k)], 1).astype(np.float32)
    sm = scenes._assemble("small_mixed", (rng2.random((nb, 3)) * 0.2 + 0.15).astype(np.float32), pos(nb), scenes._random_unit_quaternions(rng2, nb),
                          (rng2.random(nb) * 0.2 + 0.15).astype(np.float32), pos(nb))
    x = nudge_b200.Sim(sm, stream=st.cuda_stream)
    for _ in range(300):
        x.step()
    x.download_bodies()
    small = {}
    for kind in ("down", "lidar", "random"):
        for n in (65536, maxn):
            load(family(kind, n, x.transforms, rng2, abi)); timed(n)
            small["%s_%d" % (kind, n)] = round(timed(n), 4)
    res["small_mixed"] = dict(colliders=sm.n_colliders, grid_level=x.debug_scalar("ray_grid_level"), fallback_rays=x.debug_scalar("ray_fallbacks"), call_ms=small)
    res.update(card())
    print(json.dumps(res))
    x.close()


if __name__ == "__main__":
    main()
