"""What body impulses cost on the c2 pile (scenes.box_drop(65536), settled, nb_step graph replay on a created stream); DESIGN.md §8.9.

Alternating windows of the same context:
  (a) steps alone;
  (b) each step plus one nb_apply_body_impulses of 16 random bodies;
  (c) each step plus one nb_apply_radial_impulse (radius 3 around a random body);
  (d) each step plus the same 16-body edit done without this call: nb_download_bodies, a vectorised numpy edit, nb_upload_bodies.
Then the time of one call for n = 1, 1,024 and 65,536 entries (and of one radial impulse): the host clock around the call and a stream
synchronise, and CUDA events around the work it enqueues.  Prints one JSON line with the card's name, power limit and SM clock, read in the
same run.  GPU only: without a CUDA device it refuses to run.
usage: python scripts/body_impulse_cost.py [--boxes 65536] [--presim 1500] [--window 200] [--rounds 4] [--reps 50]"""
import argparse, json, os, subprocess, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
import numpy as np


def card():
    out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout
    name, power, clock, max_clock = (x.strip() for x in out.strip().splitlines()[0].split(","))
    return dict(gpu=name, power_limit=power, sm_clock=clock, max_sm_clock=max_clock)


def host_edit(x, rows):
    """The 16-body edit as an application does it without the call: download every body, edit the rows in numpy, upload every body."""
    from tests.impulse_ref import world_inverse_inertia
    x.download_bodies()
    b = rows["body"].astype(np.int64)   # distinct bodies
    m = x.properties["mass_inverse"][b][:, None]
    x.momentum["velocity"][b] += m * rows["impulse"]
    W = world_inverse_inertia(x.transforms["rotation"][b], x.properties[b])
    t = np.cross(rows["offset"], rows["impulse"]) + rows["angular_impulse"]
    M = W[:, [0, 3, 4, 3, 1, 5, 4, 5, 2]].reshape(-1, 3, 3)
    x.momentum["angular_velocity"][b] += np.einsum("nij,nj->ni", M, t).astype(np.float32)
    x.idle[b] = 0
    x.upload_bodies()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--boxes", type=int, default=65536)
    ap.add_argument("--presim", type=int, default=1500)
    ap.add_argument("--window", type=int, default=200, help="steps per timed window")
    ap.add_argument("--rounds", type=int, default=4, help="(a) / (b) / (c) / (d) window rounds")
    ap.add_argument("--reps", type=int, default=50, help="calls timed per list length")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("body_impulse_cost.py measures on a CUDA GPU (H100); there is none here and no CPU path")
    import nudge_b200
    from nudge_b200 import scenes
    from tests.impulse_ref import random_impulses
    s = scenes.box_drop(args.boxes, iterations=8, seed=2)
    B = s.n_bodies
    x = nudge_b200.Sim(s, stream=torch.cuda.Stream().cuda_stream)
    ts = torch.cuda.ExternalStream(x.stream.value)
    sync = lambda: x._ck(x.lib.nb_stream_synchronize(x.ctx, x.stream), "nb_stream_synchronize")
    for _ in range(args.presim):
        x.step()
    sync()
    rng = np.random.default_rng(1)

    def kicks():   # 16 distinct random bodies, small impulses (about 0.05 m/s), so that the pile stays the pile
        r = random_impulses(rng, np.arange(1, B), 16, scale=0.05, duplicates=False, zeros=0.0)
        r["impulse"] /= x.properties["mass_inverse"][r["body"]][:, None]
        return r

    x.download_bodies()
    blasts = [(x.transforms["position"][int(b)].copy(), 3.0, 0.5) for b in rng.integers(1, B, args.window)]
    kick_rows = []
    edits = dict(a=lambda i: None, b=lambda i: x.apply_body_impulses(kick_rows[i]), c=lambda i: x.apply_radial_impulse(*blasts[i]),
                 d=lambda i: host_edit(x, kick_rows[i]))
    rate = {k: [] for k in edits}
    for _ in range(args.rounds):
        for k, edit in edits.items():
            kick_rows[:] = [kicks() for _ in range(args.window)]
            sync()
            t0 = time.perf_counter()
            for i in range(args.window):
                edit(i)
                x.step()
            sync()
            rate[k].append(args.window / (time.perf_counter() - t0))
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
    for n in (1, 1024, 65536):
        r = random_impulses(rng, np.arange(1, B), n, scale=1e-3)
        x.apply_body_impulses(r)   # sizes the staging buffers once
        per_call["list_%d" % n] = call_times(lambda: x.apply_body_impulses(r), args.reps)
    per_call["radial"] = call_times(lambda: x.apply_radial_impulse(*blasts[0]), args.reps)
    per_call["step"] = call_times(x.step, args.reps)
    x.download_bodies()
    med = {k: float(np.median(v)) for k, v in rate.items()}
    res = dict(script="body_impulse_cost", boxes=args.boxes, presim=args.presim, window_steps=args.window, window_rounds=args.rounds,
               steps_per_s={k: [round(v, 1) for v in rate[k]] for k in rate}, median_steps_per_s={k: round(v, 1) for k, v in med.items()},
               cost_per_step_us={k: round(1e6 * (1.0 / med[k] - 1.0 / med["a"]), 1) for k in "bcd"},
               cost_pct={k: round(100.0 * (med["a"] / med[k] - 1.0), 2) for k in "bcd"},
               per_call=per_call, graph_active=graph, active_bodies=x.counts().active, finite=bool(np.isfinite(x.transforms["position"]).all()), **card())
    print(json.dumps(res))
    x.close()


if __name__ == "__main__":
    main()
