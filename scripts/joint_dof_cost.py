"""What swing-cone and twist limits cost on the c2 pile (scenes.box_drop(65536), settled, nb_step graph replay on a created stream); DESIGN.md
§8.20.

The ball joints of §8.13's set-up (chains of 8 neighbouring bodies, red-black: 2 levels), 4,096 of them at rest (rel_rotation = the rest
pose), twist axis a's x axis.  Alternating windows of the same context:
  (a) the ball joints without drives;
  (b) CONE | TWIST on every ball (cone 0.5 rad, twist range +-0.5 rad): 12,288 appended rows built and solved inside the step;
  (c) the ball joints without drives plus the same cone and twist rows built on the host every step: nb_download_bodies, the rows in
      vectorised numpy (float32, the header's formulas), then nb_upload_constraint_rows, which re-records the step's graph.
Prints one JSON line with the card's name, power limit and SM clock, read in the same run.  GPU only: without a CUDA device it refuses to run.
usage: python scripts/joint_dof_cost.py [--boxes 65536] [--presim 1500] [--window 25] [--rounds 12]"""
import argparse, json, os, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
import numpy as np
from scripts.body_impulse_cost import card
from scripts.joint_cost import qrot
from scripts.joint_drive_cost import qmul
from oracle import joints_ref

CONE, TWIST = 0.5, 0.5


def swing_twist_rows(xf, joints, dt, impulse, row_dtype):
    """The cone row and the two twist rows of every ball joint (both sides bodies), vectorised; impulse = the rows' accumulated impulses."""
    f = np.float32
    a, b = joints["a"], joints["b"]
    qa, qb = xf["rotation"][a], xf["rotation"][b]
    d = qmul(qmul(qa, joints["rel_rotation"]), qb * f([-1, -1, -1, 1])).astype(f)
    d[d[:, 3] < 0] *= -1
    u = qrot(qa, joints["axis_a"]).astype(f)
    a_ = (d[:, :3] * u).sum(1)
    sh, ch = -a_, d[:, 3]
    p = d[:, :3] - u * a_[:, None]
    ss, cs = np.sqrt((p * p).sum(1)), np.sqrt(sh * sh + ch * ch)
    st, ct = np.where(cs > 0, sh / np.where(cs > 0, cs, 1), 0), np.where(cs > 0, ch / np.where(cs > 0, cs, 1), 1)
    n = np.where(ss[:, None] > 0, p / np.where(ss > 0, ss, 1)[:, None], 0)
    k = joints["beta"] / f(dt)
    bias = lambda C: np.where(C > 0, C / f(dt), k * C)
    sc, cc, sl, cl = f(np.sin(0.5 * CONE)), f(np.cos(0.5 * CONE)), f(np.sin(-0.5 * TWIST)), f(np.cos(-0.5 * TWIST))
    rows = np.zeros((len(joints), 3), row_dtype)
    rows["a"], rows["b"] = a[:, None], b[:, None]
    rows["ang_a"][:, 0], rows["ang_b"][:, 0], rows["bias"][:, 0] = -n, n, bias(2 * (sc * cs - cc * ss))
    rows["ang_a"][:, 1], rows["ang_b"][:, 1], rows["bias"][:, 1] = -u, u, bias(2 * (st * cl - ct * sl))
    rows["ang_a"][:, 2], rows["ang_b"][:, 2], rows["bias"][:, 2] = u, -u, bias(2 * (-sl * ct - cl * st))
    rows["lo"], rows["hi"] = 0.0, np.inf
    rows = rows.reshape(-1)
    rows["impulse"] = impulse
    return rows


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
        sys.exit("joint_dof_cost.py measures on a CUDA GPU (H100); there is none here and no CPU path")
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
    joints["type"] = joints_ref.BALL; joints["a"] = pairs[:, 0]; joints["b"] = pairs[:, 1]; joints["beta"] = 0.2
    mid = 0.5 * (xf["position"][pairs[:, 0]] + xf["position"][pairs[:, 1]])
    joints["anchor_a"] = qrot(inv(qa), mid - xf["position"][pairs[:, 0]]); joints["anchor_b"] = qrot(inv(qb), mid - xf["position"][pairs[:, 1]])
    joints["axis_a"] = (1.0, 0.0, 0.0)
    rel = qmul(inv(qa), qb)
    joints["rel_rotation"] = rel / np.linalg.norm(rel, axis=1, keepdims=True)
    drives = np.zeros(len(joints), nudge_b200.JOINT_DRIVE)
    drives["joint"] = np.arange(len(joints)); drives["flags"] = nudge_b200.JOINT_CONE | nudge_b200.JOINT_TWIST
    drives["cone"], drives["lower"], drives["upper"] = CONE, -TWIST, TWIST
    drives["break_force"], drives["break_torque"] = np.inf, np.inf
    dt = float(s.time_step)
    state = dict(impulse=np.zeros(3 * len(joints), np.float32))

    def host_rows():
        x.download_bodies()
        x.upload_constraint_rows(swing_twist_rows(x.transforms, joints, dt, state["impulse"], nudge_b200.ROW))

    def setup(k):
        x.upload_joints(joints)
        x.upload_joint_drives(drives if k == "b" else None)
        if k != "c":
            x.upload_constraint_rows(np.zeros(0, nudge_b200.ROW))
    edits = dict(a=lambda: None, b=lambda: None, c=host_rows)
    rate = {k: [] for k in edits}
    records = {}
    for _ in range(args.rounds):
        for k, edit in edits.items():
            setup(k)
            edit(); x.step()   # a changed drive or row set re-records the graph outside the window
            sync()
            r0 = x.debug_scalar("graph_records")
            t0 = time.perf_counter()
            for i in range(args.window):
                edit()
                x.step()
                if k == "c":
                    state["impulse"] = x.download_constraint_rows(3 * len(joints))["impulse"]
            sync()
            rate[k].append(args.window / (time.perf_counter() - t0))
            records[k] = records.get(k, 0) + x.debug_scalar("graph_records") - r0
    x.download_bodies()
    med = {k: float(np.median(v)) for k, v in rate.items()}
    res = dict(script="joint_dof_cost", boxes=args.boxes, presim=args.presim, window_steps=args.window, window_rounds=args.rounds, joints=len(joints),
               joint_levels=int(joints_ref.joint_levels(joints).max()) + 1, steps_per_s={k: [round(v, 1) for v in rate[k]] for k in rate},
               median_steps_per_s={k: round(v, 1) for k, v in med.items()}, cost_per_step_us={k: round(1e6 * (1.0 / med[k] - 1.0 / med["a"]), 1) for k in "bc"},
               records_inside_windows=records, finite=bool(np.isfinite(x.transforms["position"]).all()), **card())
    print(json.dumps(res))
    x.close()


if __name__ == "__main__":
    main()
