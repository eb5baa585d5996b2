"""What contact events cost on the c2 pile (scenes.box_drop(65536), settled, nb_step graph replay on a created stream); DESIGN.md §8.5.

Reports, as one JSON line:
  - steps/s in alternating windows with events off and on (the three extra launches per step);
  - events per step, and the drain (nb_download_contact_events) time per call after the step has finished;
  - steps/s of an application loop that drains every step, and of the same loop done the other way: nb_download_contacts
    (every contact row and sleeping pair over PCIe) plus a host diff of the pair keys against the previous step;
  - the card's name and power limit, read in the same run.
GPU only: without a CUDA device it refuses to run.
usage: python scripts/contact_events_cost.py [--boxes 65536] [--presim 900] [--window 200] [--pairs 5]"""
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
    ap.add_argument("--pairs", type=int, default=5, help="off / on window pairs")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("contact_events_cost.py measures on a CUDA GPU (H100); there is none here and no CPU path")
    import nudge_b200
    from nudge_b200 import scenes
    s = scenes.box_drop(args.boxes, iterations=8, seed=2)
    stream = torch.cuda.Stream()
    g = nudge_b200.Sim(s, stream=stream.cuda_stream)
    sync = lambda: g._ck(g.lib.nb_stream_synchronize(g.ctx, g.stream), "nb_stream_synchronize")
    for _ in range(args.presim):
        g.step()
    sync()
    cap = 1 << 20

    def timed(loop, steps):
        sync(); t0 = time.perf_counter()
        for _ in range(steps):
            loop()
        sync()
        return steps / (time.perf_counter() - t0)

    off, on, events = [], [], 0
    for _ in range(args.pairs):
        g.enable_contact_events(0); g.step()          # the toggle re-records the graph: one untimed step
        off.append(timed(g.step, args.window))
        g.enable_contact_events(cap); g.step()
        on.append(timed(g.step, args.window))
        events += len(g.contact_events()[0])          # the first step after the toggle included
    # drain every step: the application loop of a game
    drains = []

    def step_and_drain():
        g.step()
        sync()   # the drain alone, not the step it would otherwise wait for
        t0 = time.perf_counter(); ev, _ = g.contact_events(); drains.append(time.perf_counter() - t0)
    drain_rate = timed(step_and_drain, args.window)
    # the same loop without events: every contact and sleeping pair to the host, diffed there
    g.enable_contact_events(0); g.step()
    prev = [np.zeros(0, np.uint64)]
    diff_events, downloads, diffs = [], [], []

    def step_and_diff():
        g.step()
        sync()
        t0 = time.perf_counter()
        g.download_contacts()
        t1 = time.perf_counter()
        cur = np.unique(g.contact_tags[:g.contacts.count])
        asleep = g.sleeping_pairs[:g.contacts.sleeping_count]
        begin = np.setdiff1d(cur, prev[0], assume_unique=True)
        end = np.setdiff1d(np.setdiff1d(prev[0], cur, assume_unique=True), asleep)
        diff_events.append(len(begin) + len(end))
        prev[0] = np.union1d(cur, np.intersect1d(prev[0], asleep))
        downloads.append(t1 - t0); diffs.append(time.perf_counter() - t1)
    step_and_diff()
    diff_events.clear(); downloads.clear(); diffs.clear()
    host_rate = timed(step_and_diff, args.window)
    c = g.counts()
    res = dict(script="contact_events_cost", boxes=args.boxes, presim=args.presim, window_steps=args.window, window_pairs=args.pairs,
               contacts=int(c.contacts), sleeping_pairs=int(c.sleeping),
               steps_per_s_events_off=[round(x, 1) for x in off], steps_per_s_events_on=[round(x, 1) for x in on],
               median_off=round(float(np.median(off)), 1), median_on=round(float(np.median(on)), 1),
               cost_pct=round(100.0 * (np.median(off) / np.median(on) - 1.0), 2),
               events_per_step=round(events / (args.pairs * (args.window + 1)), 2),
               drain_ms_median=round(1e3 * float(np.median(drains)), 4), steps_per_s_drain_every_step=round(drain_rate, 1),
               steps_per_s_download_contacts_and_host_diff=round(host_rate, 1), host_diff_events_per_step=round(float(np.mean(diff_events)), 2),
               download_contacts_ms_median=round(1e3 * float(np.median(downloads)), 3), host_diff_ms_median=round(1e3 * float(np.median(diffs)), 3),
               bytes_per_step_download_contacts=int(c.contacts) * (32 + 8 + 8 + 4) + int(c.sleeping) * 8,
               **card())
    print(json.dumps(res))
    g.close()


if __name__ == "__main__":
    main()
