"""What body states cost on the c2 pile (scenes.box_drop(65536), settled, nb_step graph replay on a created stream); DESIGN.md §8.19.

Alternating windows of the same context:
  (a) steps alone;
  (b) each step after one nb_set_body_states of 1,024 random bodies (NB_BODY_POSE | NB_BODY_VELOCITY) through device pointers: the rows
      live in a CUDA tensor, gathered once at the start, so every step puts those bodies back where they were (a reset);
  (c) each step after the same edit done without the call: nb_download_bodies, a numpy edit of the 1,024 rows, nb_upload_bodies.
(a) against (b) is the step rate with and without the set; the step graph's record count is read before and after, to show it is kept.
Then the time of one call: the set of 1,024 (device pointers) and the host round trip; a gather of every body into a CUDA tensor, against
nb_download_transforms + nb_download_momentum + a copy of both to the device.  Host clock around the call and a stream synchronise, and CUDA
events around the work.  Prints one JSON line with the card's name, power limit and SM clock, read in the same run.  GPU only.
usage: python scripts/body_state_cost.py [--boxes 65536] [--presim 1500] [--window 200] [--rounds 4] [--reps 50] [--n 1024]"""
import argparse, ctypes, json, os, subprocess, sys, time
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
    ap.add_argument("--rounds", type=int, default=4, help="(a) / (b) / (c) window rounds")
    ap.add_argument("--reps", type=int, default=50, help="calls timed per case")
    ap.add_argument("--n", type=int, default=1024, help="bodies per set")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("body_state_cost.py measures on a CUDA GPU (H100); there is none here and no CPU path")
    import nudge_b200
    from nudge_b200 import abi, scenes
    s = scenes.box_drop(args.boxes, iterations=8, seed=2)
    B = s.n_bodies
    x = nudge_b200.Sim(s, stream=torch.cuda.Stream().cuda_stream)
    ts = torch.cuda.ExternalStream(x.stream.value)
    sync = lambda: x._ck(x.lib.nb_stream_synchronize(x.ctx, x.stream), "nb_stream_synchronize")
    for _ in range(args.presim):
        x.step()
    sync()
    rng = np.random.default_rng(1)
    bodies = rng.choice(np.arange(1, B), args.n, replace=False).astype(np.uint32)
    rows = x.get_body_states(bodies)
    rows["velocity"] = 0; rows["angular_velocity"] = 0
    t_rows = torch.from_numpy(rows.view(np.int32).reshape(-1).copy()).cuda()
    t_skip = torch.zeros(1, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    fields = abi.BODY_POSE | abi.BODY_VELOCITY
    set_dev = lambda: x.set_body_states(None, fields, device_ptrs=(t_rows.data_ptr(), t_skip.data_ptr()), n=args.n)
    b64 = bodies.astype(np.int64)

    def set_host():   # the edit as an application does it without the call
        x.download_bodies()
        x.transforms["position"][b64] = rows["position"]; x.transforms["rotation"][b64] = rows["rotation"]
        x.momentum["velocity"][b64] = 0; x.momentum["angular_velocity"][b64] = 0; x.idle[b64] = 0
        x.upload_bodies()

    set_dev(); sync()   # sizes the set's scratch once
    records = x.debug_scalar("graph_records")
    edits = dict(a=None, b=set_dev, c=set_host)
    rate = {k: [] for k in edits}
    for _ in range(args.rounds):
        for k, edit in edits.items():
            sync()
            t0 = time.perf_counter()
            for i in range(args.window):
                if edit is not None:
                    edit()
                x.step()
            sync()
            rate[k].append(args.window / (time.perf_counter() - t0))
    records_after = x.debug_scalar("graph_records")
    graph = x.debug_scalar("graph_active")

    def call_times(fn, reps):
        host, dev = [], []
        for _ in range(reps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            sync(); torch.cuda.synchronize()
            t0 = time.perf_counter()
            e0.record(ts); fn(); e1.record(ts)
            sync(); torch.cuda.synchronize()
            host.append(1e6 * (time.perf_counter() - t0))
            dev.append(1e3 * e0.elapsed_time(e1))
        return dict(host_us=round(float(np.median(host)), 1), device_us=round(float(np.median(dev)), 1))

    out = torch.zeros(B * 16, dtype=torch.int32, device="cuda")
    xf = abi.aligned_array(B, scenes.TRANSFORM); mom = abi.aligned_array(B, scenes.MOMENTUM)
    t_xf = torch.zeros(B * 8, dtype=torch.int32, device="cuda"); t_mom = torch.zeros(B * 8, dtype=torch.int32, device="cuda")
    vp = lambda a: ctypes.c_void_p(a.ctypes.data)

    def gather_dev():
        x.get_body_states(device_ptrs=(0, out.data_ptr()), n=B)

    def gather_host():   # the read as an application does it without the call: whole prefixes to the host, then to the device
        x._ck(x.lib.nb_download_transforms(x.ctx, vp(xf), B, x.stream), "nb_download_transforms")
        x._ck(x.lib.nb_download_momentum(x.ctx, vp(mom), B, x.stream), "nb_download_momentum")
        sync()
        with torch.cuda.stream(ts):
            t_xf.copy_(torch.from_numpy(xf.view(np.int32).reshape(-1)), non_blocking=False)
            t_mom.copy_(torch.from_numpy(mom.view(np.int32).reshape(-1)), non_blocking=False)

    per_call = dict(set_device=call_times(set_dev, args.reps), set_host_round_trip=call_times(set_host, args.reps),
                    gather_device=call_times(gather_dev, args.reps), gather_host_round_trip=call_times(gather_host, args.reps),
                    step=call_times(x.step, args.reps))
    gather_dev(); sync()
    got = out.cpu().numpy().view(abi.BODY_STATE)
    x.download_bodies()
    same = bool(got["position"].tobytes() == np.ascontiguousarray(x.transforms["position"]).tobytes())
    med = {k: float(np.median(v)) for k, v in rate.items()}
    res = dict(script="body_state_cost", boxes=args.boxes, presim=args.presim, window_steps=args.window, window_rounds=args.rounds, n=args.n,
               steps_per_s={k: [round(v, 1) for v in rate[k]] for k in rate}, median_steps_per_s={k: round(v, 1) for k, v in med.items()},
               cost_per_step_us={k: round(1e6 * (1.0 / med[k] - 1.0 / med["a"]), 1) for k in "bc"},
               cost_pct={k: round(100.0 * (med["a"] / med[k] - 1.0), 2) for k in "bc"},
               per_call=per_call, graph_active=graph, graph_records_before=records, graph_records_after=records_after,
               gather_equals_download=same, skipped=int(t_skip.item()), finite=bool(np.isfinite(x.transforms["position"]).all()), **card())
    print(json.dumps(res))
    x.close()


if __name__ == "__main__":
    main()
