"""What joints cost on the c2 pile (scenes.box_drop(65536), settled, nb_step graph replay on a created stream); DESIGN.md §8.13.

Alternating windows of the same context:
  (a) steps without joints;
  (b) steps with 4,096 ball joints resident (chains of 8 neighbouring bodies, each chain's joints ordered red-black: 2 joint levels);
  (c) the same joints as 12,288 user rows rebuilt on the host every step: nb_download_bodies, the rows in vectorised numpy, then
      nb_upload_constraint_rows, which re-records the step's graph.
Then the time of one nb_upload_joints of the 4,096 joints (same structure: the graph is kept): the host clock around the call and a stream
synchronise.  Prints one JSON line with the card's name, power limit and SM clock, read in the same run.  GPU only: without a CUDA device
it refuses to run.
usage: python scripts/joint_cost.py [--boxes 65536] [--presim 1500] [--window 25] [--rounds 12] [--reps 50]"""
import argparse, json, os, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
import numpy as np
from scripts.body_impulse_cost import card
from oracle import joints_ref


def qrot(q, v):
    t = 2.0 * np.cross(q[:, :3], v)
    return v + q[:, 3:4] * t + np.cross(q[:, :3], t)


def ball_rows(xf, joints, dt, impulse, row_dtype):
    """The 3 rows of every ball joint (both sides bodies), vectorised; impulse = the rows' accumulated impulses."""
    a, b = joints["a"], joints["b"]
    ra = qrot(xf["rotation"][a], joints["anchor_a"]); rb = qrot(xf["rotation"][b], joints["anchor_b"])
    err = (xf["position"][a] + ra) - (xf["position"][b] + rb)
    rows = np.zeros((len(joints), 3), row_dtype)
    eye = np.eye(3, dtype=np.float32)
    for k in range(3):
        rows["a"][:, k], rows["b"][:, k] = a, b
        rows["lin_a"][:, k] = eye[k]; rows["ang_a"][:, k] = np.cross(ra, eye[k])
        rows["lin_b"][:, k] = -eye[k]; rows["ang_b"][:, k] = -np.cross(rb, eye[k])
        rows["bias"][:, k] = joints["beta"] / np.float32(dt) * err[:, k]
    rows["lo"], rows["hi"] = -np.inf, np.inf
    rows = rows.reshape(-1)
    rows["impulse"] = impulse
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--boxes", type=int, default=65536)
    ap.add_argument("--presim", type=int, default=1500)
    ap.add_argument("--window", type=int, default=25, help="steps per timed window (short windows, alternated, so that the pile evolving under the steps affects every leg alike)")
    ap.add_argument("--rounds", type=int, default=12, help="(a) / (b) / (c) window rounds")
    ap.add_argument("--reps", type=int, default=50, help="nb_upload_joints calls timed")
    ap.add_argument("--joints", type=int, default=4096)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("joint_cost.py measures on a CUDA GPU (H100); there is none here and no CPU path")
    import nudge_b200
    from nudge_b200 import scenes
    s = scenes.box_drop(args.boxes, iterations=8, seed=2)
    x = nudge_b200.Sim(s, stream=torch.cuda.Stream().cuda_stream)
    sync = lambda: x._ck(x.lib.nb_stream_synchronize(x.ctx, x.stream), "nb_stream_synchronize")
    for _ in range(args.presim):
        x.step()
    x.download_bodies()
    # chains of 8 bodies neighbouring in x (sorted by position), anchors midway so that the joints start at rest; per chain the joints
    # (0,1) (2,3) (4,5) (6,7) first, then (1,2) (3,4) (5,6): every joint of the first half is independent of the others, likewise the second
    order = 1 + np.lexsort((x.transforms["position"][1:, 2], x.transforms["position"][1:, 0]))
    chains = order[:len(order) // 8 * 8].reshape(-1, 8)[:(args.joints + 6) // 7]
    pairs = np.concatenate([chains[:, [k, k + 1]] for k in (0, 2, 4, 6, 1, 3, 5)])[:args.joints]
    joints = np.zeros(len(pairs), nudge_b200.JOINT)
    joints["type"] = 0; joints["a"] = pairs[:, 0]; joints["b"] = pairs[:, 1]; joints["beta"] = 0.2; joints["rel_rotation"][:, 3] = 1.0
    xf = x.transforms
    mid = 0.5 * (xf["position"][pairs[:, 0]] + xf["position"][pairs[:, 1]])
    inv = lambda q: q * np.float32([-1, -1, -1, 1])
    joints["anchor_a"] = qrot(inv(xf["rotation"][pairs[:, 0]]), mid - xf["position"][pairs[:, 0]])
    joints["anchor_b"] = qrot(inv(xf["rotation"][pairs[:, 1]]), mid - xf["position"][pairs[:, 1]])
    dt = float(s.time_step)
    state = dict(impulse=np.zeros(3 * len(joints), np.float32))

    def host_rows():
        x.download_bodies()
        x.upload_constraint_rows(ball_rows(x.transforms, joints, dt, state["impulse"], nudge_b200.ROW))

    def setup(k):
        x.upload_joints(joints if k == "b" else None)
        if k != "c":
            x.upload_constraint_rows(np.zeros(0, nudge_b200.ROW))
    edits = dict(a=lambda: None, b=lambda: None, c=host_rows)
    rate = {k: [] for k in edits}
    for _ in range(args.rounds):
        for k, edit in edits.items():
            setup(k)
            edit(); x.step()   # a changed joint set re-records the graph outside the window
            sync()
            t0 = time.perf_counter()
            for i in range(args.window):
                edit()
                x.step()
                if k == "c":
                    state["impulse"] = x.download_constraint_rows(3 * len(joints))["impulse"]
            sync()
            rate[k].append(args.window / (time.perf_counter() - t0))
    x.upload_joints(joints); x.upload_constraint_rows(np.zeros(0, nudge_b200.ROW))
    x.step(); sync()
    records = x.debug_scalar("graph_records")
    host = []
    for _ in range(args.reps):
        sync()
        t0 = time.perf_counter()
        x.upload_joints(joints)
        sync()
        host.append(1e6 * (time.perf_counter() - t0))
    x.step(); sync()
    kept = x.debug_scalar("graph_records") == records
    x.download_bodies()
    med = {k: float(np.median(v)) for k, v in rate.items()}
    res = dict(script="joint_cost", boxes=args.boxes, presim=args.presim, window_steps=args.window, window_rounds=args.rounds, joints=len(joints),
               chains=len(chains), joint_levels=int(joints_ref.joint_levels(joints).max()) + 1, steps_per_s={k: [round(v, 1) for v in rate[k]] for k in rate}, median_steps_per_s={k: round(v, 1) for k, v in med.items()},
               cost_per_step_us={k: round(1e6 * (1.0 / med[k] - 1.0 / med["a"]), 1) for k in "bc"},
               upload_joints_host_us=round(float(np.median(host)), 1), graph_kept_by_reupload=bool(kept), graph_active=x.debug_scalar("graph_active"),
               finite=bool(np.isfinite(x.transforms["position"]).all()), **card())
    print(json.dumps(res))
    x.close()


if __name__ == "__main__":
    main()
