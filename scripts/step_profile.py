#!/usr/bin/env python
"""Per-kernel breakdown of one nb_step on a settled bench.py scene (a development aid, not part of the library).

  python scripts/step_profile.py --out DIR [--config c2] [--solver parity|throughput] [--steps 20]

Settles the scene the way bench.py does, times `--steps` graph replays of nb_step with CUDA events (L2 flushed between steps,
profiler off), then replays the same number of steps under torch.profiler with CUDA activities in a run of its own.  Writes
DIR/kernels.csv (kernel, launches per step, µs per step), DIR/summary.json (card, power limit, step time, summed kernel time and
the difference: the idle time between graph nodes, contacts, and the box-box pairs that survived the face SAT and went to k_np_clip)
and prints the table."""
import argparse, csv, json, os, subprocess, sys
from collections import defaultdict

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
CNT_SURV = 40   # position of CNT_SURV in the device counters (the enum at the top of nudge_b200/csrc/nb_collide.cuh)


def card():
    q = "name,power.limit,clocks.max.sm,driver_version"
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
        return dict(zip(q.split(","), [x.strip() for x in out.split(",")]))
    except Exception as e:  # noqa: BLE001
        return {"error": repr(e)[:200]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--config", default="c2")
    ap.add_argument("--solver", default="parity", choices=["parity", "throughput"])
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--presim", type=int, default=-1)
    args = ap.parse_args()
    import numpy as np
    import torch
    import nudge_b200
    from bench import CONFIGS, settle_gpu
    from nudge_b200 import scenes

    cfg = CONFIGS[args.config]
    side = torch.cuda.Stream()
    torch.cuda.set_stream(side)
    ns = argparse.Namespace(iterations=0, boxes=65536)
    scene = scenes.box_drop(65536, iterations=8, seed=2) if args.config == "c2" else cfg["scene"](ns, 1)
    sim = nudge_b200.Sim(scene, stream=side.cuda_stream)
    if args.solver == "throughput":
        sim.set_solver_mode("throughput")
    settle_gpu(sim, cfg["presim"] if args.presim < 0 else args.presim)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    K = args.steps
    for _ in range(5):
        sim.step()

    # step time without the profiler, the way bench.py takes it
    E = lambda: torch.cuda.Event(enable_timing=True)
    ev = [(E(), E()) for _ in range(K)]
    torch.cuda.synchronize()
    l0 = sim.launch_count()
    for k in range(K):
        flush.fill_(k & 255)
        ev[k][0].record(); sim.step(); ev[k][1].record()
    torch.cuda.synchronize()
    launches = (sim.launch_count() - l0) / K
    step_us = 1e3 * sum(a.elapsed_time(b) for a, b in ev) / K

    os.makedirs(args.out, exist_ok=True)
    trace = os.path.join(args.out, "step.pt.trace.json")
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for k in range(K):
            flush.fill_(k & 255)
            sim.step()
        torch.cuda.synchronize()
    prof.export_chrome_trace(trace)
    events = json.load(open(trace))["traceEvents"]
    per = defaultdict(lambda: [0, 0.0])
    for e in events:
        if e.get("ph") != "X" or e.get("cat") not in ("kernel", "gpu_memset", "gpu_memcpy"):
            continue
        name = e["name"]
        if e["cat"] == "kernel" and ("fill" in name.lower() or "FillFunctor" in name):
            continue   # the L2 flush between steps
        if e["cat"] != "kernel":
            name = "[%s] %s" % (e["cat"], name)
        short = name.split("(")[0].replace("void ", "")
        per[short][0] += 1
        per[short][1] += float(e["dur"])
    rows = sorted(((n, c / K, us / K) for n, (c, us) in per.items()), key=lambda r: -r[2])
    kernel_us = sum(r[2] for r in rows)
    with open(os.path.join(args.out, "kernels.csv"), "w", newline="") as f:
        w = csv.writer(f)
        w.writerow(["kernel", "launches_per_step", "us_per_step"])
        for n, c, us in rows:
            w.writerow([n, "%.2f" % c, "%.2f" % us])
    summary = {"card": card(), "config": args.config, "solver": args.solver, "steps": K, "contacts": int(sim.counts().contacts),
               "clip_survivors": int(sim.debug("counts", np.uint32)[CNT_SURV]),
               "library_launches_per_step": launches, "traced_ops_per_step": sum(r[1] for r in rows),
               "step_us_graph_replay": step_us, "kernel_us_per_step": kernel_us, "idle_between_nodes_us": step_us - kernel_us,
               "note": "step_us from CUDA events without the profiler; kernel_us from the profiler's trace of the same number of replays"}
    json.dump(summary, open(os.path.join(args.out, "summary.json"), "w"), indent=1)
    os.remove(trace)
    print(json.dumps(summary))
    print("%-48s %9s %10s" % ("kernel", "launches", "us/step"))
    for n, c, us in rows:
        print("%-48s %9.2f %10.2f" % (n[:48], c, us))
    sim.close()


if __name__ == "__main__":
    main()
