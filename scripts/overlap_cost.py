"""What overlap queries cost on the c2 pile (scenes.box_drop(65536), settled, nb_step graph replay on a created stream); DESIGN.md §8.15.

  (a) calls of 1, 1,024 and 65,536 queries with device pointers: spheres of radius 1.5 around body centres, and oriented boxes (random unit
      rotations, half extents 0.5 to 1.5) around body centres; CUDA events, median of --reps calls, with the hits per query;
  (b) a few large queries (spheres and boxes spanning the pile), which test every collider;
  (c) the host alternative for 1,024 sphere queries: nb_download_bodies, then oracle/overlap_ref.py's numpy brute force, and whether it
      gives the same bytes as the device;
  (d) nb_step alone against nb_step plus one 1,024-sphere-query call per step, alternating windows.
Prints one JSON line with the card's name, power limit and SM clock, read in the same run.  GPU only: without a CUDA device it refuses.
usage: python scripts/overlap_cost.py [--presim 1500] [--reps 20] [--window 25] [--rounds 8]"""
import argparse, json, os, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
import numpy as np
from scripts.body_impulse_cost import card


def family(kind, n, xf, rng, abi):
    p = xf["position"][1:]
    q = np.zeros(n, abi.OVERLAP_QUERY)
    q["mask"] = 0xffffffff; q["ignore_body"] = abi.RAY_NO_HIT; q["rotation"][:, 3] = 1.0
    q["center"] = p[rng.integers(0, len(p), n)]
    if kind == "sphere":
        q["shape"] = abi.OVERLAP_SPHERE; q["radius"] = 1.5
    elif kind == "box":
        v = rng.normal(size=(n, 4)); v /= np.linalg.norm(v, axis=1, keepdims=True)
        q["shape"] = abi.OVERLAP_BOX; q["rotation"] = v; q["half_extents"] = rng.uniform(0.5, 1.5, (n, 3))
    else:   # large: spheres and boxes spanning the pile
        lo, hi = p.min(axis=0), p.max(axis=0)
        q["center"] = 0.5 * (lo + hi); q["shape"][1::2] = abi.OVERLAP_BOX
        q["radius"] = 0.5 * float(np.linalg.norm(hi - lo)); q["half_extents"] = 0.5 * (hi - lo)
    return q


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
        sys.exit("overlap_cost.py measures on a CUDA GPU (H100); there is none here and no CPU path")
    import nudge_b200
    from nudge_b200 import abi, scenes
    from oracle import overlap_ref, raycast_ref
    st = torch.cuda.Stream()
    x = nudge_b200.Sim(scenes.box_drop(args.boxes, iterations=8, seed=2), stream=st.cuda_stream)
    for _ in range(args.presim):
        x.step()
    x.download_bodies()
    rng = np.random.default_rng(1)
    maxn, cap = 65536, 1 << 24
    d_q = torch.zeros(maxn * 64, dtype=torch.uint8, device="cuda")
    d_h = torch.zeros(cap * 16, dtype=torch.uint8, device="cuda")
    d_o = torch.zeros(maxn + 1, dtype=torch.int32, device="cuda")
    ptrs = (d_q.data_ptr(), d_h.data_ptr(), d_o.data_ptr())

    def timed(n):
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        ms = []
        for _ in range(args.reps):
            ev[0].record(st)
            x.overlap(None, capacity=cap, device_ptrs=ptrs, n=n)
            ev[1].record(st)
            ev[1].synchronize()
            ms.append(ev[0].elapsed_time(ev[1]))
        return float(np.median(ms))

    def load(q):
        d_q[:len(q) * 64].copy_(torch.from_numpy(q.view(np.uint8).copy()))
        torch.cuda.synchronize()

    res = dict(script="overlap_cost", boxes=args.boxes, presim=args.presim, reps=args.reps, call_ms={}, hits_per_query={})
    for kind, sizes in (("sphere", (1, 1024, maxn)), ("box", (1, 1024, maxn)), ("large", (4,))):
        for n in sizes:
            load(family(kind, n, x.transforms, rng, abi)); timed(n)
            res["call_ms"]["%s_%d" % (kind, n)] = round(timed(n), 4)
            res["hits_per_query"]["%s_%d" % (kind, n)] = round(int(d_o[n].item()) / n, 2)
    res["fallbacks"] = x.debug_scalar("overlap_fallbacks")
    q = family("sphere", 1024, x.transforms, rng, abi)
    t0 = time.perf_counter()
    x.download_bodies()
    want = overlap_ref.query(raycast_ref.Scene.of_sim(x), q)
    res["host_1024_sphere_ms"] = round(1e3 * (time.perf_counter() - t0), 1)
    got = x.overlap(q)
    res["host_equals_device"] = bool(got[0].tobytes() == want[0].tobytes() and got[1].tobytes() == want[1].tobytes())
    load(q)
    rate = {"step": [], "step_plus_1024_queries": []}
    for _ in range(args.rounds):
        for k in rate:
            st.synchronize()
            t0 = time.perf_counter()
            for _ in range(args.window):
                x.step()
                if k != "step":
                    x.overlap(None, capacity=cap, device_ptrs=ptrs, n=1024)
            st.synchronize()
            rate[k].append(args.window / (time.perf_counter() - t0))
    res["steps_per_s"] = {k: [round(v, 1) for v in rate[k]] for k in rate}
    res["median_steps_per_s"] = {k: round(float(np.median(v)), 1) for k, v in rate.items()}
    res.update(card())
    print(json.dumps(res))
    x.close()


if __name__ == "__main__":
    main()
