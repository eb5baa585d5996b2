"""What joint springs cost on the c2 pile (scenes.box_drop(65536), settled, nb_step graph replay on a created stream); DESIGN.md §8.21.

The joints of §8.13's set-up (chains of 8 neighbouring bodies, red-black: 2 levels), as 4,096 hinges about the world z axis at rest.
Alternating windows of the same context:
  (a) the hinges without springs;
  (b) a spring on every hinge (stiffness 20, damping 2, max_force 50) with a new target for every joint uploaded before every step (the
      graph is kept);
  (c) the host PD way without springs: every step nb_download_bodies, the hinge angles and rates and the torques
      k * (target - theta) - c * theta_dot in numpy, and nb_upload_constraint_rows of one hinge-Jacobian row per joint holding that
      torque's impulse (lo = hi = impulse).
Prints one JSON line with the card's name, power limit and SM clock, read in the same run.  GPU only: without a CUDA device it refuses to run.
usage: python scripts/joint_spring_cost.py [--boxes 65536] [--presim 1500] [--window 25] [--rounds 12]"""
import argparse, json, os, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
import numpy as np
from scripts.body_impulse_cost import card
from scripts.joint_cost import qrot
from scripts.joint_drive_cost import qmul
from oracle import joints_ref

K, C, F = 20.0, 2.0, 50.0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--boxes", type=int, default=65536)
    ap.add_argument("--presim", type=int, default=1500)
    ap.add_argument("--window", type=int, default=25, help="steps per timed window (short windows, alternated, so that the pile evolving under the steps affects every leg alike)")
    ap.add_argument("--rounds", type=int, default=12, help="(a) / (b) / (c) window rounds")
    ap.add_argument("--joints", type=int, default=4096)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("joint_spring_cost.py measures on a CUDA GPU (H100); there is none here and no CPU path")
    import nudge_b200
    from nudge_b200 import scenes
    s = scenes.box_drop(args.boxes, iterations=8, seed=2)
    x = nudge_b200.Sim(s, stream=torch.cuda.Stream().cuda_stream)
    sync = lambda: x._ck(x.lib.nb_stream_synchronize(x.ctx, x.stream), "nb_stream_synchronize")
    for _ in range(args.presim):
        x.step()
    x.download_bodies()
    order = 1 + np.lexsort((x.transforms["position"][1:, 2], x.transforms["position"][1:, 0]))
    chains = order[:len(order) // 8 * 8].reshape(-1, 8)[:(args.joints + 6) // 7]
    pairs = np.concatenate([chains[:, [k, k + 1]] for k in (0, 2, 4, 6, 1, 3, 5)])[:args.joints]
    xf = x.transforms
    qa, qb = xf["rotation"][pairs[:, 0]].astype(np.float64), xf["rotation"][pairs[:, 1]].astype(np.float64)
    inv = lambda q: q * np.array([-1, -1, -1, 1])
    joints = np.zeros(len(pairs), nudge_b200.JOINT)
    joints["type"] = joints_ref.HINGE; joints["a"] = pairs[:, 0]; joints["b"] = pairs[:, 1]; joints["beta"] = 0.2
    mid = 0.5 * (xf["position"][pairs[:, 0]] + xf["position"][pairs[:, 1]])
    joints["anchor_a"] = qrot(inv(qa), mid - xf["position"][pairs[:, 0]]); joints["anchor_b"] = qrot(inv(qb), mid - xf["position"][pairs[:, 1]])
    z = np.tile([0.0, 0.0, 1.0], (len(pairs), 1))
    joints["axis_a"] = qrot(inv(qa), z); joints["axis_b"] = qrot(inv(qb), z)
    rel = qmul(inv(qa), qb)
    joints["rel_rotation"] = rel / np.linalg.norm(rel, axis=1, keepdims=True)
    springs = np.zeros(len(joints), nudge_b200.JOINT_SPRING)
    springs["joint"] = np.arange(len(joints)); springs["stiffness"], springs["damping"], springs["max_force"] = K, C, F
    dt = np.float32(s.time_step)
    rng = np.random.default_rng(1)
    rows = np.zeros(len(joints), nudge_b200.ROW)
    rows["a"], rows["b"] = joints["a"], joints["b"]

    def targets():
        springs["target"][:, 0] = rng.uniform(-0.5, 0.5, len(springs)).astype(np.float32)
        x.upload_joint_springs(springs)

    def host_pd():
        x.download_bodies()
        t = x.transforms["rotation"]
        qa, qb = t[joints["a"]].astype(np.float64), t[joints["b"]].astype(np.float64)
        d = qmul(qmul(qa, joints["rel_rotation"].astype(np.float64)), inv(qb))
        u = qrot(qa, joints["axis_a"].astype(np.float64))
        theta = 2.0 * np.arctan2(-(d[:, :3] * u).sum(1) * np.sign(d[:, 3] + 1e-30), np.abs(d[:, 3]))
        w = x.momentum["angular_velocity"].astype(np.float64)
        rate = ((w[joints["b"]] - w[joints["a"]]) * u).sum(1)
        tau = np.clip(K * (rng.uniform(-0.5, 0.5, len(joints)) - theta) - C * rate, -F, F)
        rows["ang_a"], rows["ang_b"] = -u, u
        rows["lo"] = rows["hi"] = rows["impulse"] = (tau * float(dt)).astype(np.float32)
        x.upload_constraint_rows(rows)

    edits = dict(a=lambda: None, b=targets, c=host_pd)
    rate = {k: [] for k in edits}
    records = {}
    for _ in range(args.rounds):
        for k, edit in edits.items():
            x.upload_joints(joints)
            x.upload_joint_springs(springs if k == "b" else None)
            x.upload_constraint_rows(rows if k == "c" else rows[:0])
            edit(); x.step()   # a changed spring or row set re-records the graph outside the window
            sync()
            r0 = x.debug_scalar("graph_records")
            t0 = time.perf_counter()
            for i in range(args.window):
                edit()
                x.step()
            sync()
            rate[k].append(args.window / (time.perf_counter() - t0))
            records[k] = records.get(k, 0) + x.debug_scalar("graph_records") - r0
    x.download_bodies()
    med = {k: float(np.median(v)) for k, v in rate.items()}
    res = dict(script="joint_spring_cost", boxes=args.boxes, presim=args.presim, window_steps=args.window, window_rounds=args.rounds, joints=len(joints),
               joint_levels=int(joints_ref.joint_levels(joints).max()) + 1, steps_per_s={k: [round(v, 1) for v in rate[k]] for k in rate},
               median_steps_per_s={k: round(v, 1) for k, v in med.items()}, cost_per_step_us={k: round(1e6 * (1.0 / med[k] - 1.0 / med["a"]), 1) for k in "bc"},
               records_inside_windows=records,
               finite=bool(np.isfinite(x.transforms["position"]).all()), **card())
    print(json.dumps(res))
    x.close()


if __name__ == "__main__":
    main()
