"""What sensor colliders cost on the c2 pile (scenes.box_drop(65536), settled, nb_step graph replay on a created stream); DESIGN.md §8.7.

Two contexts are settled the same way: (g) the plain pile and (h) the same pile with 48 static sensor zones on the ground among the boxes
(tests/sensor_ref.add_sensors).  Sensors exert no force, so both step the same bodies bit for bit.  Reports, as one JSON line:
  - steps/s in alternating windows of (a) g without a table, (b) g with an all-zero table (the sensor launches run, no pair is a sensor
    pair) and (c) h with its zones (thousands of overlapping sensor pairs);
  - (h)'s candidate sensor pairs and overlaps per step, and whether g and h ended with the same transforms;
  - the summed device time of the k_sensor_* kernels per step of (c), from torch.profiler in a separate, untimed run;
  - the card's name, power limit and SM clock, read in the same run.
GPU only: without a CUDA device it refuses to run.
usage: python scripts/sensor_cost.py [--boxes 65536] [--presim 1500] [--window 200] [--rounds 5]"""
import argparse, json, os, subprocess, sys, time
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
    ap.add_argument("--window", type=int, default=200, help="steps per timed window")
    ap.add_argument("--rounds", type=int, default=5, help="(a) / (b) / (c) window rounds")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("sensor_cost.py measures on a CUDA GPU (H100); there is none here and no CPU path")
    import nudge_b200
    from nudge_b200 import scenes
    from tests.sensor_ref import add_sensors
    s = scenes.box_drop(args.boxes, iterations=8, seed=2)
    L = 15.0 * np.sqrt(args.boxes / 8191.0)
    zones = [((x, 2.0, z), (4.5, 2.0, 4.5)) for x in np.linspace(-0.8 * L, 0.8 * L, 8) for z in np.linspace(-0.8 * L, 0.8 * L, 6)]
    z = add_sensors(s, zones=zones)
    g = nudge_b200.Sim(s, stream=torch.cuda.Stream().cuda_stream)
    h = nudge_b200.Sim(z, stream=torch.cuda.Stream().cuda_stream)
    sync = lambda x: x._ck(x.lib.nb_stream_synchronize(x.ctx, x.stream), "nb_stream_synchronize")
    for x in (g, h):
        for _ in range(args.presim):
            x.step()
        sync(x)
    g.download_bodies(); h.download_bodies()
    same = g.transforms.tobytes() == h.transforms.tobytes()

    def timed(x, steps):
        sync(x)
        t0 = time.perf_counter()
        for _ in range(steps):
            x.step()
        sync(x)
        return steps / (time.perf_counter() - t0)

    zero = np.zeros(s.n_colliders, np.uint8)
    a, b, c, launches, cand, hits = [], [], [], {}, [], []
    for _ in range(args.rounds):
        g.upload_sensors(None); g.step()                           # a table change re-records the graph: one untimed step
        a.append(timed(g, args.window))
        k = g.launch_count(); g.step(); launches["a"] = g.launch_count() - k
        g.upload_sensors(zero); g.step()
        b.append(timed(g, args.window))
        k = g.launch_count(); g.step(); launches["b"] = g.launch_count() - k
        c.append(timed(h, args.window))
        k = h.launch_count(); h.step(); launches["c"] = h.launch_count() - k
        cand.append(len(h.debug("sensor_pairs", np.uint64))); hits.append(len(h.sensor_overlaps()))
    from torch.profiler import profile, ProfilerActivity
    steps = 20
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            h.step_staged()
        sync(h)
    sensor_us = sum(e.device_time_total for e in prof.key_averages() if e.key.startswith("k_sensor")) / steps
    med = lambda v: round(float(np.median(v)), 1)
    res = dict(script="sensor_cost", boxes=args.boxes, zones=len(zones), presim=args.presim, window_steps=args.window, window_rounds=args.rounds,
               steps_per_s_no_table=[round(x, 1) for x in a], steps_per_s_all_zero=[round(x, 1) for x in b], steps_per_s_zones=[round(x, 1) for x in c],
               median_no_table=med(a), median_all_zero=med(b), median_zones=med(c),
               all_zero_cost_pct=round(100.0 * (np.median(a) / np.median(b) - 1.0), 2), zones_cost_pct=round(100.0 * (np.median(a) / np.median(c) - 1.0), 2),
               candidate_sensor_pairs=cand, overlaps=hits, same_transforms_after_presim=same, launches_per_step=launches,
               sensor_kernels_us_per_step=round(sensor_us, 1), **card())
    print(json.dumps(res))
    g.close(); h.close()


if __name__ == "__main__":
    main()
