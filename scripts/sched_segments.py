#!/usr/bin/env python
"""How well the batch scheduler's replay splits into segments on a settled bench.py scene (a development aid).

  python scripts/sched_segments.py --out DIR [--config c2]

Settles the scene the way bench.py does, reads the tag-ordered body pairs the scheduler replays (nb_debug_read "cab"), and replays
them with the plain-Python restatement in tests/sched_ref.py.  Prints the number of buckets the device's segmented replay sent
to the sequential one; per bucket, the distribution of the gaps between the contacts after which the slot list is empty; for 8,
16, 32 and 64 segments per bucket, the lengths of the joins on the chain of picked runs (contacts a join replays before it couples
with a speculative run) and the number of buckets that would fall back to the sequential replay; and the same for 32 segments
with one speculative run per segment instead of eight.  --device-only stops after the device's count (scenes too large for the
Python replay).  Writes the same to DIR/sched_segments.json and DIR/sched_segments.txt."""
import argparse, json, os, sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--config", default="c2")
    ap.add_argument("--cap", type=int, default=64, help="list positions a segment run may hold before its bucket falls back")
    ap.add_argument("--device-only", action="store_true", help="only the device's count of buckets that fell back (large scenes)")
    args = ap.parse_args()
    import numpy as np
    import torch
    import nudge_b200
    from bench import CONFIGS, settle_gpu
    from nudge_b200 import scenes
    from tests import sched_ref

    cfg = CONFIGS[args.config]
    side = torch.cuda.Stream()
    torch.cuda.set_stream(side)
    ns = argparse.Namespace(iterations=0, boxes=65536)
    scene = scenes.box_drop(65536, iterations=8, seed=2) if args.config == "c2" else cfg["scene"](ns, 1)
    sim = nudge_b200.Sim(scene, stream=side.cuda_stream)
    settle_gpu(sim, cfg["presim"])
    sim.step()
    torch.cuda.synchronize()
    cab = sim.debug("cab", np.uint32).reshape(-1, 2)
    n = len(cab)
    fb_dev = sim.debug_scalar("sched_fallback")
    lines = ["config %s: %d contacts, %d per bucket; buckets the device's segmented replay sent to the sequential one: %d" %
             (args.config, n, (n + 15) // 16, fb_dev)]
    out = {"config": args.config, "contacts": n, "sched_fallback": fb_dev, "gaps": {}, "segments": {}}
    if args.device_only:
        print(lines[0])
        return

    bs = sched_ref.buckets(cab)
    allgaps = []
    for k, p in enumerate(bs):
        ea = set()
        sched_ref.replay(p, 0, len(p), [], [None] * len(p), {}, empty_after=ea)
        pts = np.array(sorted(ea)) if ea else np.zeros(0, np.int64)
        gaps = np.diff(np.concatenate([[-1], pts])) if len(pts) else np.array([len(p)])
        allgaps.append(gaps)
        q = np.percentile(gaps, [50, 90, 99, 100]).tolist()
        out["gaps"][k] = {"empty_points": int(len(pts)), "p50": q[0], "p90": q[1], "p99": q[2], "max": q[3]}
        lines.append("bucket %2d: %6d contacts, list empty after %6d of them; gap p50 %5.0f p90 %5.0f p99 %5.0f max %6.0f" %
                     (k, len(p), len(pts), *q))
    g = np.concatenate(allgaps)
    lines.append("all buckets: gap p50 %.0f p90 %.0f p99 %.0f max %.0f" % tuple(np.percentile(g, [50, 90, 99, 100])))

    ref_batch, ref_lane = sched_ref.schedule_sequential(cab)
    nbmax = (n + 15) // 16
    for w in (8, 16, 32, 64):
        seg_len = (nbmax + w - 1) // w
        stats = {}
        batch, lane, fb = sched_ref.schedule_segmented(cab, w, seg_len, cap=args.cap, stats=stats)
        jl = np.array(stats.get("join_len", [0]))
        same = bool((batch == ref_batch).all() and (lane == ref_lane).all())
        out["segments"][w] = {"seg_len": seg_len, "fallback_buckets": int(fb), "joins": int(len(stats.get("join_len", []))),
                              "join_mean": float(jl.mean()), "join_p90": float(np.percentile(jl, 90)), "join_max": int(jl.max()),
                              "same_schedule": same}
        lines.append("W=%2d: segment %5d contacts, %3d joins, join length mean %.1f p90 %.0f max %d, %d buckets fall back, schedule %s" %
                     (w, seg_len, len(stats.get("join_len", [])), jl.mean(), np.percentile(jl, 90), jl.max(), fb,
                      "identical" if same else "DIFFERENT"))
    seg_len = (nbmax + 31) // 32
    _, _, fb1 = sched_ref.schedule_segmented(cab, 32, seg_len, cap=args.cap, phases=1)
    out["one_phase_w32_fallback_buckets"] = int(fb1)
    lines.append("W=32 with one speculative run per segment (from the segment start only): %d buckets fall back" % fb1)
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "sched_segments.json"), "w") as f:
        json.dump(out, f, indent=1)
    with open(os.path.join(args.out, "sched_segments.txt"), "w") as f:
        f.write("\n".join(lines) + "\n")
    print("\n".join(lines))


if __name__ == "__main__":
    main()
