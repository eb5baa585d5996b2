"""What continuous collision costs (nb_upload_ccd_bodies; DESIGN.md §8.18), nb_step graph replay on a created stream.

  (a) the c2 pile (scenes.box_drop(65536), settled): steps/s in alternating windows with no set, with 1,024 listed bodies and with every
      body listed at threshold 0 (the worst case: every awake body casts every step), each body's sphere at 0.95 of its box's smallest half
      extent; the launches per step and the clamps and fallbacks of the last step of each leg;
  (b) the bullet scene: 256 boxes of half extent 0.1 fired at 120 m/s at a 0.2-thick static wall (dt = 1/60), steps/s without and with the
      set over the first 120 steps, and whether any box centre ends beyond the wall.
Prints one JSON line with the card's name, power limit and SM clock, read in the same run.  GPU only: without a CUDA device it refuses.
usage: python scripts/ccd_cost.py [--presim 1500] [--window 50] [--rounds 6]"""
import argparse, json, os, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
import numpy as np
from scripts.body_impulse_cost import card


def rows(abi, bodies, radius):
    e = np.zeros(len(bodies), abi.CCD_BODY)
    e["body"], e["radius"], e["category"], e["mask"] = bodies, radius, 0xffff, 0xffff
    return e


def bullet_scene(scenes):
    """rows x cols boxes of half extent 0.1 at x = -10.9 just above the ground, at 120 m/s along +x, and a static wall at x = 0."""
    y, z = np.meshgrid(-9.85 + 0.25 * np.arange(4), -9.6 + 0.3 * np.arange(64), indexing="ij")
    pos = np.stack([np.full(256, -10.9), y.ravel(), z.ravel()], 1).astype(np.float32)
    s = scenes._assemble("bullets", np.full((256, 3), 0.1, np.float32), pos, None, np.zeros(0, np.float32), np.zeros((0, 3), np.float32))
    s.box_tags = np.append(s.box_tags, np.uint32(s.n_boxes))
    wd = np.zeros(1, scenes.BOX); wd["size"] = (0.1, 20.0, 20.0)
    wt = np.zeros(1, scenes.TRANSFORM); wt["rotation"][0, 3] = 1.0; wt["position"] = (0.0, -10.0, 0.0)
    s.box_data = np.concatenate([s.box_data, wd]); s.box_transforms = np.concatenate([s.box_transforms, wt])
    s.momentum["velocity"][1:] = (120.0, 0.0, 0.0)
    s.time_step = np.float32(1.0 / 60.0)
    return s


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--boxes", type=int, default=65536)
    ap.add_argument("--presim", type=int, default=1500)
    ap.add_argument("--window", type=int, default=50, help="steps per timed window")
    ap.add_argument("--rounds", type=int, default=6)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("ccd_cost.py measures on a CUDA GPU (H100); there is none here and no CPU path")
    import nudge_b200
    from nudge_b200 import abi, scenes
    x = nudge_b200.Sim(scenes.box_drop(args.boxes, iterations=8, seed=2), stream=torch.cuda.Stream().cuda_stream)
    sync = lambda s: s._ck(s.lib.nb_stream_synchronize(s.ctx, s.stream), "nb_stream_synchronize")
    for _ in range(args.presim):
        x.step()
    sync(x)
    B = x.scene.n_bodies
    radius = 0.95 * x.scene.box_data["size"][1:B].min(axis=1)   # body k carries box k (box 0 is the ground)
    rng = np.random.default_rng(1)
    some = np.sort(rng.choice(np.arange(1, B), 1024, replace=False))
    legs = {"no_set": None, "listed_1024": rows(abi, some, radius[some - 1]), "every_body": rows(abi, np.arange(1, B), radius)}

    def timed(s, steps):
        sync(s)
        t0 = time.perf_counter()
        for _ in range(steps):
            s.step()
        sync(s)
        return steps / (time.perf_counter() - t0)

    rate = {k: [] for k in legs}
    launches, clamps = {}, {}
    for _ in range(args.rounds):
        for k, e in legs.items():
            x.upload_ccd_bodies(e)
            x.step()   # records the leg's graph outside the window
            rate[k].append(timed(x, args.window))
            c0 = x.launch_count(); x.step(); launches[k] = x.launch_count() - c0
            if e is not None:
                clamps[k] = int((x.debug("ccd_hits", np.uint32).reshape(-1, 2)[:, 1] != abi.RAY_NO_HIT).sum())
    fallbacks = x.debug_scalar("ccd_fallbacks")
    active = x.counts().active
    x.close()
    med = lambda v: round(float(np.median(v)), 1)
    res = dict(script="ccd_cost", boxes=args.boxes, presim=args.presim, window_steps=args.window, rounds=args.rounds,
               steps_per_s={k: [round(v, 1) for v in r] for k, r in rate.items()}, median_steps_per_s={k: med(r) for k, r in rate.items()},
               cost_ms_per_step={k: round(1e3 / med(rate[k]) - 1e3 / med(rate["no_set"]), 4) for k in legs if k != "no_set"},
               launches_per_step=launches, clamped_last_step=clamps, ccd_fallbacks=fallbacks, active_bodies=active)
    # (b) the bullet scene
    bullets = {}
    for k in ("no_set", "set"):
        s = bullet_scene(scenes)
        b = nudge_b200.Sim(s, stream=torch.cuda.Stream().cuda_stream)
        if k == "set":
            b.upload_ccd_bodies(rows(abi, np.arange(1, s.n_bodies), 0.09))
        b.step(); b.step()   # the graph's record and a first replay outside the timing
        r = timed(b, 118)
        b.download_bodies()
        bullets[k] = dict(steps_per_s=round(r, 1), beyond_wall=int((b.transforms["position"][1:, 0] > 0.1).sum()))
        b.close()
    res["bullets"] = bullets
    res.update(card())
    print(json.dumps(res))


if __name__ == "__main__":
    main()
