# compute-sanitizer passes over a small scene (SURVEY.md section 5): memcheck (global/shared out-of-bounds, misaligned, leaks of the
# relaxed 128-bit token words and bulk copies) and racecheck (shared-memory hazards: sort tiles, scheduler slots, TMA stage ring).
# usage: bash scripts/sanitize.sh   (on the GPU box; writes gpurun_out/sanitize_*.log)
mkdir -p gpurun_out
cat > /tmp/nb_sanitize_case.py <<'PY'
import numpy as np, nudge_b200
from nudge_b200 import scenes
s = scenes.demo_scene(96, 96, iterations=4, spread=2.0, height=8.0)
g = nudge_b200.Sim(s)
g.enable_contact_events(4096)   # the event kernels run inside nb_write_cached_impulses
for _ in range(6): g.step_staged()
g.set_solver_mode("throughput")
for _ in range(4): g.step_staged()
st = g.get_body_states([1, 5, 9, 5]); g.get_body_states()   # body states: host mode, then device mode below
st["position"][:, 1] += 0.5
g.set_body_states(st, 3); g.set_body_states(st, 2)
import torch
t_idx = torch.tensor([1, 5, 9, 5], dtype=torch.int32, device="cuda"); t_out = torch.zeros(64, dtype=torch.int32, device="cuda")
t_skip = torch.zeros(1, dtype=torch.int32, device="cuda")
torch.cuda.synchronize()
g.get_body_states(device_ptrs=(t_idx.data_ptr(), t_out.data_ptr()), n=4)
g.set_body_states(None, 3, device_ptrs=(t_out.data_ptr(), t_skip.data_ptr()), n=4)
g.step_staged()
g.get_body_contact_impulses(); g.get_body_contact_impulses([0, 3, 3]); g.get_contact_pair_impulses(0.0)   # contact impulse reports
t_cb = torch.zeros(8 * s.n_bodies, dtype=torch.int32, device="cuda"); t_cp = torch.zeros(12 * 64, dtype=torch.int32, device="cuda")
torch.cuda.synchronize()
g.get_body_contact_impulses(device_ptrs=(t_idx.data_ptr(), t_cb.data_ptr()), n=4)
g.get_contact_pair_impulses(device_ptrs=(t_cp.data_ptr(), t_skip.data_ptr()), capacity=64)
ev, dropped = g.contact_events()
c = g.counts(); print("contacts", c.contacts, "overflow", c.overflow, "events", len(ev), "dropped", dropped)
PY
for tool in memcheck racecheck; do
  timeout 900 compute-sanitizer --tool $tool --error-exitcode 9 env PYTHONPATH=$PWD python /tmp/nb_sanitize_case.py > gpurun_out/sanitize_$tool.log 2>&1
  echo "$tool rc=$? $(grep -E 'ERROR SUMMARY|RACECHECK SUMMARY' gpurun_out/sanitize_$tool.log | tail -1)"
done
