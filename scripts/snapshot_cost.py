"""What device-resident snapshots cost on the c2 pile (scenes.box_drop(65536), settled, nb_step graph replay on a created stream); DESIGN.md
section 8.12.

  (a) one nb_snapshot_save and one nb_snapshot_restore: CUDA events around each call, median over --reps;
  (b) the live bytes one copy moves (what the state file of the same state holds, plus the snapshot's count words), and the bandwidth that
      is as a share of the H100's 3.35 TB/s data-sheet HBM bandwidth (a copy reads and writes each byte once);
  (c) a rollback of 8 steps (restore, then 8 graph-replayed steps) against 8 plain steps, alternated over --rounds;
  (d) nb_save_state + nb_load_state of the same state through a temporary file: the host clock around the pair.
Also the device memory of one snapshot for this context, from the element sizes and capacities.  Prints one JSON line with the card's name,
power limit and SM clock, read in the same run.  GPU only: without a CUDA device it refuses to run.
usage: python scripts/snapshot_cost.py [--boxes 65536] [--presim 1500] [--reps 50] [--rounds 24]"""
import argparse, json, os, sys, tempfile, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
import numpy as np
from scripts.body_impulse_cost import card

HBM_BYTES_PER_S = 3.35e12


def snapshot_bytes(cfg_bodies, cfg_boxes, cfg_spheres, cfg_conn, cfg_contacts):
    """The arena of nb_snapshot_create: every section at its capacity, padded to 16 bytes (DESIGN.md section 8.12)."""
    pad = lambda n: (n + 15) // 16 * 16
    K = cfg_boxes + cfg_spheres
    sizes = [32 * cfg_bodies, 16 * cfg_bodies, 32 * cfg_bodies, cfg_bodies, 4 * cfg_boxes, 16 * cfg_boxes, 32 * cfg_boxes, 4 * cfg_spheres,
             4 * cfg_spheres, 32 * cfg_spheres, 8 * cfg_conn, 8 * cfg_contacts, 4 * cfg_contacts, 16 * cfg_contacts, 4 * K, K, 0, 48 * cfg_bodies,
             cfg_bodies, 8 * cfg_conn]
    return sum(pad(n) for n in sizes) + 16


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--boxes", type=int, default=65536)
    ap.add_argument("--presim", type=int, default=1500)
    ap.add_argument("--reps", type=int, default=50, help="saves and restores timed")
    ap.add_argument("--rounds", type=int, default=24, help="rollback / plain rounds of 8 steps")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("snapshot_cost.py measures on a CUDA GPU (H100); there is none here and no CPU path")
    import nudge_b200
    from nudge_b200 import scenes
    s = scenes.box_drop(args.boxes, iterations=8, seed=2)
    x = nudge_b200.Sim(s, stream=torch.cuda.Stream().cuda_stream)
    ts = torch.cuda.ExternalStream(x.stream.value)
    sync = lambda: x._ck(x.lib.nb_stream_synchronize(x.ctx, x.stream), "nb_stream_synchronize")
    for _ in range(args.presim):
        x.step()
    sync()
    c = x.counts()
    snap = x.snapshot()
    sync()

    def timed(call):
        out = []
        for _ in range(args.reps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(ts); call(); e1.record(ts)
            e1.synchronize()
            out.append(1e3 * e0.elapsed_time(e1))
        return float(np.median(out))

    save_us = timed(lambda: x.snapshot(into=snap))
    restore_us = timed(lambda: x.restore(snap))
    B, nb, ns = s.n_bodies, s.n_boxes, s.n_spheres
    live = B * (32 + 16 + 32 + 1) + nb * (4 + 16 + 32) + ns * (4 + 4 + 32) + 8 * len(s.connections) + c.cache * (8 + 4 + 16) + 12

    def window(rollback):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(ts)
        if rollback:
            x.restore(snap)
        for _ in range(8):
            x.step()
        e1.record(ts)
        e1.synchronize()
        return 1e3 * e0.elapsed_time(e1)

    x.snapshot(into=snap)
    window(True); window(False)   # warm: the graph is recorded
    roll, plain = [], []
    for _ in range(args.rounds):
        roll.append(window(True)); plain.append(window(False))
    x.restore(snap); sync()
    with tempfile.TemporaryDirectory() as d:
        p = os.path.join(d, "s.nbstate")
        files = []
        for _ in range(5):
            t0 = time.perf_counter(); x.save_state(p); x.load_state(p); sync(); files.append(1e6 * (time.perf_counter() - t0))
        file_bytes = os.path.getsize(p)
    cfg = (s.n_bodies, s.n_boxes, s.n_spheres, max(1, len(s.connections)), x.cap)
    res = dict(card(), workload="c2 pile: %d bodies, %d cache entries, settled after %d steps" % (B, c.cache, args.presim),
               save_us=round(save_us, 1), restore_us=round(restore_us, 1), live_bytes=live,
               save_hbm_share=round(2 * live / (save_us * 1e-6) / HBM_BYTES_PER_S, 3), restore_hbm_share=round(2 * live / (restore_us * 1e-6) / HBM_BYTES_PER_S, 3),
               rollback8_us=round(float(np.median(roll)), 1), plain8_us=round(float(np.median(plain)), 1),
               state_file_save_load_us=round(float(np.median(files)), 1), state_file_bytes=file_bytes,
               snapshot_device_bytes=snapshot_bytes(*cfg))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
