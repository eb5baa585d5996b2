"""What the warm start costs inside the exact-order solver on the c2 pile (scenes.box_drop(65536), settled); DESIGN.md section 2.8.

From one snapshot of the settled pile, alternated over --rounds:
  (a) nb_step with its launches made one by one (NB_GRAPH=0): the k_solve launch of the step, which follows k_warm_start;
  (b) the staged calls (nb_setup_contact_constraints does the warm start, then nb_apply_impulses(8)): the k_solve launch of the sweeps.
Both k_solve times come from the library's CUDA events around that launch (nb_debug_timing).  (a) - (b) is what the warm start adds to
the step's solver launch: 80 us while it was a dependency-chained pass inside k_solve, about zero since k_warm_start.  Prints one JSON
line with the card's name, power limit and SM clock, read in the same run.  GPU only: without a CUDA device it refuses to run.
usage: python scripts/warm_start_cost.py [--boxes 65536] [--presim 900] [--rounds 20]"""
import argparse, json, os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
import numpy as np
from scripts.body_impulse_cost import card


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--boxes", type=int, default=65536)
    ap.add_argument("--presim", type=int, default=900)
    ap.add_argument("--rounds", type=int, default=20)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("warm_start_cost.py measures on a CUDA GPU (H100); there is none here and no CPU path")
    os.environ["NB_GRAPH"] = "0"   # read by nb_create: nb_step makes its launches one by one, so the timing events see them
    import nudge_b200
    from nudge_b200 import scenes
    s = scenes.box_drop(args.boxes, iterations=8, seed=2)
    x = nudge_b200.Sim(s, stream=torch.cuda.Stream().cuda_stream)
    sync = lambda: x._ck(x.lib.nb_stream_synchronize(x.ctx, x.stream), "nb_stream_synchronize")
    for _ in range(args.presim):
        x.step()
    sync()
    snap = x.snapshot()
    c = x.counts()

    def solve_ms(staged):
        x.restore(snap)
        x.timing_enable(True)
        x.step_staged() if staged else x.step()
        n, ms = x.timing()
        x.timing_enable(False)
        assert n == 1, n
        return ms

    solve_ms(False); solve_ms(True)   # warm
    step, staged = [], []
    for _ in range(args.rounds):
        step.append(solve_ms(False)); staged.append(solve_ms(True))
    x.restore(snap); sync()
    us = lambda v: round(1e3 * float(np.median(v)), 1)
    res = dict(card(), workload="c2 pile: %d bodies, %d contacts, %d batches, settled after %d steps" % (s.n_bodies, c.contacts, c.batches, args.presim),
               rounds=args.rounds, k_solve_in_step_us=us(step), k_solve_staged_us=us(staged), difference_us=us(np.array(step) - np.array(staged)),
               k_solve_in_step_range_us=[us([min(step)]), us([max(step)])], k_solve_staged_range_us=[us([min(staged)]), us([max(staged)])])
    print(json.dumps(res))
    x.close()


if __name__ == "__main__":
    main()
