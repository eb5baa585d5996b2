"""What kinematic bodies cost on the c2 pile (scenes.box_drop(65536), settled, nb_step graph replay on a created stream); DESIGN.md §8.8.

Three contexts are settled the same way: (a) the plain pile, (b) the same pile with its ground moved onto a kinematic body at rest
(tests/kinematic_ref.with_kinematic_ground; the same bodies bit for bit, indices mapped) and (c) that kinematic ground rising at 0.05 m/s
after the settling, so the pile stays awake.  Reports, as one JSON line:
  - steps/s in alternating windows of (a), (b) and (c), and the launches per step of each;
  - the dependency depth of the exact Gauss-Seidel order (scripts/solver_depth.py's count) and the apply_impulses time of one step of (c),
    against the same state with the rising ground as a zero-mass DYNAMIC body instead (the workaround without kinematic bodies: every
    contact on the ground joins that body's chain);
  - the card's name, power limit and SM clock, read in the same run.
GPU only: without a CUDA device it refuses to run.
usage: python scripts/kinematic_cost.py [--boxes 65536] [--presim 1500] [--window 200] [--rounds 5]"""
import argparse, json, os, subprocess, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
import numpy as np


def card():
    out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout
    name, power, clock, max_clock = (x.strip() for x in out.strip().splitlines()[0].split(","))
    return dict(gpu=name, power_limit=power, sm_clock=clock, max_sm_clock=max_clock)


def depth(a, b, sweeps):
    """scripts/solver_depth.py's count: the longest chain of dependent contact applications over `sweeps` sweeps in slot order; body 0 and a
    side with NB_READ_ONLY (bit 31, a kinematic body) are never waited for."""
    last = {}
    for _ in range(sweeps):
        for x, y in zip(a, b):
            x = 0 if x >> 31 else x
            y = 0 if y >> 31 else y
            l = max(last.get(x, 0) if x else 0, last.get(y, 0) if y else 0) + 1
            if x: last[x] = l
            if y: last[y] = l
    return max(last.values()) if last else 0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--boxes", type=int, default=65536)
    ap.add_argument("--presim", type=int, default=1500)
    ap.add_argument("--window", type=int, default=200, help="steps per timed window")
    ap.add_argument("--rounds", type=int, default=5, help="(a) / (b) / (c) window rounds")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("kinematic_cost.py measures on a CUDA GPU (H100); there is none here and no CPU path")
    import nudge_b200
    from nudge_b200 import scenes
    from tests.kinematic_ref import with_kinematic_ground
    s = scenes.box_drop(args.boxes, iterations=8, seed=2)
    ks, k = with_kinematic_ground(s)
    rising = np.array([(k, (0.0, 0.05, 0.0), (0.0, 0.0, 0.0), 0)], scenes.KINEMATIC)
    ctx = {n: nudge_b200.Sim(x, stream=torch.cuda.Stream().cuda_stream) for n, x in (("a", s), ("b", ks), ("c", ks))}
    sync = lambda x: x._ck(x.lib.nb_stream_synchronize(x.ctx, x.stream), "nb_stream_synchronize")
    for x in ctx.values():
        for _ in range(args.presim):
            x.step()
        sync(x)
    ctx["c"].upload_kinematic_bodies(rising)
    for _ in range(50):
        ctx["c"].step()
    ctx["a"].download_bodies(); ctx["b"].download_bodies()
    rows = np.array([k] + list(range(1, k)), np.int64)
    same = ctx["a"].transforms.tobytes() == ctx["b"].transforms[rows].tobytes()

    def timed(x, steps):
        sync(x)
        t0 = time.perf_counter()
        for _ in range(steps):
            x.step()
        sync(x)
        return steps / (time.perf_counter() - t0)

    rate = {n: [] for n in ctx}
    launches = {}
    for _ in range(args.rounds):
        for n, x in ctx.items():
            rate[n].append(timed(x, args.window))
            c0 = x.launch_count(); x.step(); launches[n] = x.launch_count() - c0
    awake = {n: x.counts().active for n, x in ctx.items()}

    # one staged step of (c) and of the zero-mass dynamic ground from the same state: dependency depth and apply_impulses time
    c = ctx["c"]
    c.download_bodies(); c.download_cache()
    w_scene = ks.copy(); w_scene.kinematic = None
    w_scene.transforms[:] = c.transforms; w_scene.momentum[:] = c.momentum; w_scene.idle[:] = c.idle
    w = nudge_b200.Sim(w_scene, stream=torch.cuda.Stream().cuda_stream)
    n = c.cache.count
    w.cache_tags[:n] = c.cache_tags[:n]; w.cache_features[:n] = c.cache_features[:n]; w.cache_data[:n] = c.cache_data[:n]; w.cache.count = n
    w.upload_cache()

    def one_step(x):
        x.collide(); x.apply_gravity_damping(); x.read_cached_impulses(); x.setup_contact_constraints()
        used = np.nonzero(x.debug("row_contact", np.uint32) != 0xffffffff)[0]
        a = x.debug("row_a", np.uint32)[used].tolist(); b = x.debug("row_b", np.uint32)[used].tolist()
        sync(x)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s0 = torch.cuda.ExternalStream(x.stream.value)
        e0.record(s0); x.apply_impulses(8); e1.record(s0)
        x.update_cached_impulses(); x.write_cached_impulses(); x.advance()
        sync(x); torch.cuda.synchronize()
        return dict(depth=depth(a, b, 8), slots=len(a), batches=x.counts().batches, apply_impulses_ms=round(e0.elapsed_time(e1), 3))

    kin_step, dyn_step = one_step(c), one_step(w)
    med = lambda v: round(float(np.median(v)), 1)
    res = dict(script="kinematic_cost", boxes=args.boxes, presim=args.presim, window_steps=args.window, window_rounds=args.rounds,
               steps_per_s_no_set=[round(x, 1) for x in rate["a"]], steps_per_s_kinematic_ground_at_rest=[round(x, 1) for x in rate["b"]],
               steps_per_s_kinematic_ground_rising=[round(x, 1) for x in rate["c"]],
               median_no_set=med(rate["a"]), median_at_rest=med(rate["b"]), median_rising=med(rate["c"]),
               at_rest_cost_pct=round(100.0 * (np.median(rate["a"]) / np.median(rate["b"]) - 1.0), 2),
               rising_cost_pct=round(100.0 * (np.median(rate["a"]) / np.median(rate["c"]) - 1.0), 2),
               launches_per_step=launches, active_bodies=awake, same_transforms_after_presim=same,
               rising_step=kin_step, zero_mass_dynamic_ground_step=dyn_step, **card())
    print(json.dumps(res))
    for x in list(ctx.values()) + [w]:
        x.close()


if __name__ == "__main__":
    main()
