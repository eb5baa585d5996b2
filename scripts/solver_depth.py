"""Dependency depth of the exact Gauss-Seidel order vs the time the dataflow solver takes (development aid, GPU).

Also the depth the warm start had as a dataflow pass over the same slots (one pass of hops, like a sweep), and the longest body chain:
the serial walk k_warm_start does instead (no hand-offs, DESIGN.md section 2.8)."""
import sys, os
from collections import Counter
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
import nudge_b200, bench
from nudge_b200 import scenes

def depth(a, b, sweeps):
    """a, b: row_a / row_b in slot order.  A side with NB_READ_ONLY (bit 31, a kinematic body) is never waited for, like body 0."""
    a = [0 if x >> 31 else x for x in a]; b = [0 if x >> 31 else x for x in b]
    last = {}
    per_sweep = []
    for w in range(sweeps):
        for i in range(len(a)):
            la = last.get(a[i], 0) if a[i] else 0
            lb = last.get(b[i], 0) if b[i] else 0
            l = max(la, lb) + 1
            if a[i]: last[a[i]] = l
            if b[i]: last[b[i]] = l
        per_sweep.append(max(last.values()))
    return per_sweep

def longest_chain(a, b):
    n = Counter(x for x in a + b if x and not x >> 31)
    return max(n.values())

for n in [int(x) for x in sys.argv[1:]] or [16384, 65536]:
    scene = scenes.box_drop(n, iterations=8, seed=2)
    sim = nudge_b200.Sim(scene, device=0, stream=torch.cuda.current_stream().cuda_stream)
    bench.settle_gpu(sim, 900)
    E = lambda: torch.cuda.Event(enable_timing=True)
    ts = []
    for k in range(8):
        sim.collide(); sim.apply_gravity_damping(); sim.read_cached_impulses(); sim.setup_contact_constraints()
        e0, e1 = E(), E(); e0.record(); sim.apply_impulses(8); e1.record()
        if k == 7:
            sim.lib.nb_debug_enable(sim.ctx, 1) if hasattr(sim.lib, "nb_debug_enable") else None
            used = np.nonzero(sim.debug("row_contact", np.uint32) != 0xffffffff)[0]
            a = sim.debug("row_a", np.uint32)[used].tolist(); b = sim.debug("row_b", np.uint32)[used].tolist()
        sim.update_cached_impulses(); sim.write_cached_impulses(); sim.advance()
        torch.cuda.synchronize(); ts.append(e0.elapsed_time(e1))
    d = depth(a, b, 8)
    t = float(np.median(ts[2:]))
    print("boxes %d slots %d depth/sweep %d total-depth(8) %d apply_impulses %.3f ms -> %.3f us/hop; warm start as a dataflow pass: depth %d "
          "(9 passes: %d); k_warm_start: longest chain %d" % (n, len(a), d[0], d[-1], t, 1000 * t / d[-1], d[0], depth(a, b, 9)[-1], longest_chain(a, b)), flush=True)
