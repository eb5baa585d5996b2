"""What collision filters cost on the c2 pile (scenes.box_drop(65536), settled, nb_step graph replay on a created stream); DESIGN.md §8.6.

Reports, as one JSON line:
  - steps/s in alternating windows (a) without a table and (b) with an all-pass table (every collider category 0xffff, mask 0xffff):
    the same pairs, so the difference is what the filter word costs the broadphase;
  - steps/s of (c) a table that splits the boxes into two categories that do not collide with each other (the ground collides with
    both), on a second context settled the same way, with its pairs and contacts per step next to those of (a);
  - the card's name and power limit, read in the same run.
GPU only: without a CUDA device it refuses to run.
usage: python scripts/collision_filter_cost.py [--boxes 65536] [--presim 900] [--window 200] [--pairs 5]"""
import argparse, json, os, subprocess, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
import numpy as np


def card():
    out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout
    name, power, clock = (x.strip() for x in out.strip().splitlines()[0].split(","))
    return dict(gpu=name, power_limit=power, max_sm_clock=clock)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--boxes", type=int, default=65536)
    ap.add_argument("--presim", type=int, default=900)
    ap.add_argument("--window", type=int, default=200, help="steps per timed window")
    ap.add_argument("--pairs", type=int, default=5, help="(a) / (b) / (c) window rounds")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("collision_filter_cost.py measures on a CUDA GPU (H100); there is none here and no CPU path")
    import nudge_b200
    from nudge_b200 import scenes
    s = scenes.box_drop(args.boxes, iterations=8, seed=2)
    n = s.n_colliders
    allpass = np.zeros(n, scenes.FILTER); allpass["category"] = 0xffff; allpass["mask"] = 0xffff
    split = np.zeros(n, scenes.FILTER)
    split["category"] = np.where(np.arange(n) % 2 == 0, 1, 2); split["mask"] = split["category"]
    split[0] = (3, 3)                                              # the ground collides with both halves
    g = nudge_b200.Sim(s, stream=torch.cuda.Stream().cuda_stream)
    h = nudge_b200.Sim(s, stream=torch.cuda.Stream().cuda_stream)
    for x in (g, h):
        for _ in range(args.presim):
            x.step()
        x._ck(x.lib.nb_stream_synchronize(x.ctx, x.stream), "nb_stream_synchronize")
    h.upload_collision_filters(split)

    def timed(x, steps):
        x._ck(x.lib.nb_stream_synchronize(x.ctx, x.stream), "nb_stream_synchronize")
        t0 = time.perf_counter()
        for _ in range(steps):
            x.step()
        x._ck(x.lib.nb_stream_synchronize(x.ctx, x.stream), "nb_stream_synchronize")
        return steps / (time.perf_counter() - t0)

    none, passing, splitted, per_step = [], [], [], dict(a_pairs=[], a_contacts=[], c_pairs=[], c_contacts=[])
    launches = {}
    for _ in range(args.pairs):
        g.upload_collision_filters(None); g.step()                 # a table change re-records the graph: one untimed step
        none.append(timed(g, args.window))
        c = g.counts(); per_step["a_pairs"].append(c.pairs); per_step["a_contacts"].append(c.contacts)
        k = g.launch_count(); g.step(); launches["a"] = g.launch_count() - k
        g.upload_collision_filters(allpass); g.step()
        passing.append(timed(g, args.window))
        k = g.launch_count(); g.step(); launches["b"] = g.launch_count() - k
        splitted.append(timed(h, args.window))
        c = h.counts(); per_step["c_pairs"].append(c.pairs); per_step["c_contacts"].append(c.contacts)
        k = h.launch_count(); h.step(); launches["c"] = h.launch_count() - k
    med = lambda v: round(float(np.median(v)), 1)
    res = dict(script="collision_filter_cost", boxes=args.boxes, presim=args.presim, window_steps=args.window, window_rounds=args.pairs,
               steps_per_s_no_table=[round(x, 1) for x in none], steps_per_s_all_pass=[round(x, 1) for x in passing],
               steps_per_s_two_categories=[round(x, 1) for x in splitted],
               median_no_table=med(none), median_all_pass=med(passing), median_two_categories=med(splitted),
               all_pass_cost_pct=round(100.0 * (np.median(none) / np.median(passing) - 1.0), 2),
               pairs_per_step_no_table=per_step["a_pairs"], contacts_per_step_no_table=per_step["a_contacts"],
               pairs_per_step_two_categories=per_step["c_pairs"], contacts_per_step_two_categories=per_step["c_contacts"],
               launches_per_step=launches, **card())
    print(json.dumps(res))
    g.close(); h.close()


if __name__ == "__main__":
    main()
