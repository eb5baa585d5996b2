"""What the contact impulse reports cost on the c2 pile (scenes.box_drop(65536), settled, nb_step graph replay on a created stream); DESIGN.md
§8.22.

Per call, after one step: nb_get_body_contact_impulses of every body and of 1,024 random bodies, nb_get_contact_pair_impulses of every pair,
each in host mode (into numpy, synchronised) and device mode (into CUDA tensors), against the host alternative: nb_download_contacts plus
nb_debug_read("impulses") / ("sorted") and the transforms downloaded before the step, summed in numpy by tests/contact_impulse_ref.py (the
restatement, which is also what the alternative must compute).  Host clock around the call and a stream synchronise, and CUDA events around
the work.  Then the step rate with both device calls after every step against steps alone, in alternating windows.  Prints one JSON line with
the card's name, power limit and SM clock, read in the same run.  GPU only.
usage: python scripts/contact_impulse_cost.py [--boxes 65536] [--presim 1500] [--window 200] [--rounds 4] [--reps 30] [--n 1024]"""
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
    ap.add_argument("--rounds", type=int, default=4, help="window rounds, with and without the reports")
    ap.add_argument("--reps", type=int, default=30, help="calls timed per case")
    ap.add_argument("--n", type=int, default=1024, help="bodies of the short list")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("contact_impulse_cost.py measures on a CUDA GPU (H100); there is none here and no CPU path")
    import nudge_b200
    from nudge_b200 import abi, scenes
    from tests.contact_impulse_ref import body_report, pair_report
    s = scenes.box_drop(args.boxes, iterations=8, seed=2)
    B = s.n_bodies
    x = nudge_b200.Sim(s, stream=torch.cuda.Stream().cuda_stream)
    ts = torch.cuda.ExternalStream(x.stream.value)
    sync = lambda: x._ck(x.lib.nb_stream_synchronize(x.ctx, x.stream), "nb_stream_synchronize")
    for _ in range(args.presim):
        x.step()
    sync()
    short = np.random.default_rng(1).choice(np.arange(B), args.n, replace=False).astype(np.uint32)
    t_short = torch.from_numpy(short.view(np.int32)).cuda()
    ob = torch.zeros(B * 8, dtype=torch.int32, device="cuda"); op = torch.zeros(x.cap * 12, dtype=torch.int32, device="cuda")
    oc = torch.zeros(1, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    body_dev = lambda: x.get_body_contact_impulses(device_ptrs=(None, ob.data_ptr()), n=B)
    short_dev = lambda: x.get_body_contact_impulses(device_ptrs=(t_short.data_ptr(), ob.data_ptr()), n=args.n)
    pair_dev = lambda: x.get_contact_pair_impulses(device_ptrs=(op.data_ptr(), oc.data_ptr()), capacity=x.cap)
    body_host = lambda: x.get_body_contact_impulses()
    short_host = lambda: x.get_body_contact_impulses(short)
    pair_host = lambda: x.get_contact_pair_impulses(capacity=x.cap)
    x.download_bodies()
    pos = x.transforms["position"].copy()
    x.step(); sync()
    body_dev(); pair_dev(); sync()   # allocates the scratch once

    def host_alternative():   # what an application computes without the calls: every contact and impulse to the host, summed in numpy
        x.download_contacts()
        cv = x.contacts_view()
        imp = x.debug("impulses", scenes.IMPULSE); srt = x.debug("sorted", np.uint32)
        return body_report(cv["data"], cv["bodies"], imp, pos, B), pair_report(cv["data"], cv["bodies"], cv["tags"], imp, srt)[0]

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

    per_call = dict(bodies_all_device=call_times(body_dev, args.reps), bodies_short_device=call_times(short_dev, args.reps),
                    pairs_device=call_times(pair_dev, args.reps), bodies_all_host=call_times(body_host, args.reps),
                    bodies_short_host=call_times(short_host, args.reps), pairs_host=call_times(pair_host, args.reps),
                    host_alternative=call_times(host_alternative, max(3, args.reps // 10)), step=call_times(x.step, args.reps))
    # the step the calls above read is the last one timed: check the device rows against the restatement of it
    x.download_bodies(); pos = x.transforms["position"].copy()
    x.step(); sync()
    want_b, want_p = host_alternative()
    same = bool(x.get_body_contact_impulses().tobytes() == want_b.tobytes() and x.get_contact_pair_impulses().tobytes() == want_p.tobytes())
    n_contacts, n_pairs = int(x.counts().contacts), len(want_p)
    records = x.debug_scalar("graph_records")
    modes = dict(a=None, b=lambda: (body_dev(), pair_dev()))
    rate = {k: [] for k in modes}
    for _ in range(args.rounds):
        for k, reports in modes.items():
            sync()
            t0 = time.perf_counter()
            for _ in range(args.window):
                x.step()
                if reports is not None:
                    reports()
            sync()
            rate[k].append(args.window / (time.perf_counter() - t0))
    med = {k: float(np.median(v)) for k, v in rate.items()}
    res = dict(script="contact_impulse_cost", boxes=args.boxes, presim=args.presim, contacts=n_contacts, pairs=n_pairs, n_short=args.n,
               per_call=per_call, steps_per_s={k: [round(v, 1) for v in rate[k]] for k in rate},
               median_steps_per_s={k: round(v, 1) for k, v in med.items()}, report_cost_per_step_us=round(1e6 * (1.0 / med["b"] - 1.0 / med["a"]), 1),
               graph_records_before=records, graph_records_after=x.debug_scalar("graph_records"), equals_restatement=same, **card())
    print(json.dumps(res))
    x.close()


if __name__ == "__main__":
    main()
