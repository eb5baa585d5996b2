"""What per-body forces cost on the c2 pile (scenes.box_drop(65536), settled, nb_step graph replay on a created stream); DESIGN.md §8.11.

Alternating windows of the same context:
  (a) steps without a table;
  (b) steps with a table of default entries;
  (c) steps with every body at gravity scale 0.98 and 1 % of the bodies carrying a small upward force (0.1 of their weight) and torque;
  (d) steps without a table plus the same thrust on 16 bodies through one nb_apply_body_impulses per step, for comparison.
Then the time of one nb_set_body_forces call for n = 16, 1,024 and 65,536 entries: the host clock around the call and a stream synchronise,
and CUDA events around the work it enqueues; and the same for Sim.set_body_forces, which also keeps sim.scene's mirror of the entries.
Prints one JSON line with the card's name, power limit and SM clock, read in the same run.  GPU only: without a CUDA device it refuses to run.
usage: python scripts/body_force_cost.py [--boxes 65536] [--presim 1500] [--window 25] [--rounds 24] [--reps 50]"""
import argparse, ctypes, json, os, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
import numpy as np
from scripts.body_impulse_cost import card


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--boxes", type=int, default=65536)
    ap.add_argument("--presim", type=int, default=1500)
    ap.add_argument("--window", type=int, default=25, help="steps per timed window (short windows, alternated, so that the pile evolving under the steps affects every leg alike)")
    ap.add_argument("--rounds", type=int, default=24, help="(a) / (b) / (c) / (d) window rounds")
    ap.add_argument("--reps", type=int, default=50, help="calls timed per list length")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("body_force_cost.py measures on a CUDA GPU (H100); there is none here and no CPU path")
    import nudge_b200
    from nudge_b200 import scenes
    s = scenes.box_drop(args.boxes, iterations=8, seed=2)
    B = s.n_bodies
    x = nudge_b200.Sim(s, stream=torch.cuda.Stream().cuda_stream)
    ts = torch.cuda.ExternalStream(x.stream.value)
    sync = lambda: x._ck(x.lib.nb_stream_synchronize(x.ctx, x.stream), "nb_stream_synchronize")
    for _ in range(args.presim):
        x.step()
    sync()
    rng = np.random.default_rng(1)
    g, dt = float(s.gravity), float(s.time_step)
    pushed = rng.choice(np.arange(1, B), max(1, (B - 1) // 100), replace=False)
    mass = np.zeros(B, np.float32); mass[pushed] = 1.0 / x.properties["mass_inverse"][pushed]
    busy = scenes.default_body_forces(np.arange(1, B)); busy["gravity_scale"] = 0.98
    sel = busy["body"].searchsorted(pushed)
    busy["force"][sel, 1] = 0.1 * g * mass[pushed]; busy["torque"][sel] = (0.0, 0.05, 0.0)
    thrust16 = pushed[:16]
    kicks = np.zeros(16, scenes.BODY_IMPULSE); kicks["body"] = thrust16; kicks["impulse"][:, 1] = 0.1 * g * mass[thrust16] * dt

    def setup(k):
        if k in ("a", "d"):
            x.clear_body_forces()
        elif k == "b":
            x.clear_body_forces(); x.set_body_forces(None)
        else:
            x.clear_body_forces(); x.set_body_forces(busy)
    edits = dict(a=lambda: None, b=lambda: None, c=lambda: None, d=lambda: x.apply_body_impulses(kicks))
    rate = {k: [] for k in edits}
    active = {}
    for _ in range(args.rounds):
        for k, edit in edits.items():
            setup(k)
            edit(); x.step()   # a new table re-records the graph outside the window
            sync()
            t0 = time.perf_counter()
            for i in range(args.window):
                edit()
                x.step()
            sync()
            rate[k].append(args.window / (time.perf_counter() - t0))
            active[k] = x.counts().active
    graph = x.debug_scalar("graph_active")

    def call_times(fn, reps):
        host, dev = [], []
        for _ in range(reps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            sync()
            t0 = time.perf_counter()
            e0.record(ts); fn(); e1.record(ts)
            sync()
            host.append(1e6 * (time.perf_counter() - t0))
            dev.append(1e3 * e0.elapsed_time(e1))
        return dict(host_us=round(float(np.median(host)), 1), device_us=round(float(np.median(dev)), 1))

    per_call = {}
    for n in (16, 1024, 65536):
        r = np.ascontiguousarray(scenes.default_body_forces(rng.choice(np.arange(1, B), min(n, B - 1), replace=False))); r["gravity_scale"] = 0.98
        x.set_body_forces(r)   # sizes the staging rows once
        ptr = r.ctypes.data_as(ctypes.c_void_p)
        per_call["set_%d" % n] = call_times(lambda: x._ck(x.lib.nb_set_body_forces(x.ctx, ptr, len(r), x.stream), "nb_set_body_forces"), args.reps)
        per_call["sim_set_%d" % n] = call_times(lambda: x.set_body_forces(r), max(5, args.reps // 5))
    per_call["step"] = call_times(x.step, args.reps)
    x.download_bodies()
    med = {k: float(np.median(v)) for k, v in rate.items()}
    res = dict(script="body_force_cost", boxes=args.boxes, presim=args.presim, window_steps=args.window, window_rounds=args.rounds, pushed_bodies=len(pushed),
               steps_per_s={k: [round(v, 1) for v in rate[k]] for k in rate}, median_steps_per_s={k: round(v, 1) for k, v in med.items()},
               cost_per_step_us={k: round(1e6 * (1.0 / med[k] - 1.0 / med["a"]), 1) for k in "bcd"},
               cost_pct={k: round(100.0 * (med["a"] / med[k] - 1.0), 2) for k in "bcd"},
               active_bodies_after_window=active, per_call=per_call, graph_active=graph, finite=bool(np.isfinite(x.transforms["position"]).all()), **card())
    print(json.dumps(res))
    x.close()


if __name__ == "__main__":
    main()
