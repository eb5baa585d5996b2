"""nb_launch_count against what the device ran: every kernel the library launches increments the counter (include/nudge_b200.h), so over a
window of library calls the counter's delta equals the number of kernel records torch.profiler's CUDA activity trace holds for the window.
Cases: the staged calls and nb_step in both solver modes, plain launches and graph replays, a step with every optional stage (contact
events, sensors, a kinematic set, a body-force table, user rows), and the editing calls.  No torch op runs inside a window."""
import json
import re
import numpy as np
import pytest
import torch
import nudge_b200
from nudge_b200 import scenes
from tests.gpu_util import side_stream

pytestmark = pytest.mark.gpu
LIBRARY_KERNEL = re.compile(r"^(void )?k_\w+")


def _scene():
    return scenes.demo_scene(400, 400, iterations=4, spread=6.0, height=10.0, seed=7)


def _window(sim, calls, tmp_path):
    """Runs calls() under the profiler; returns (nb_launch_count delta, names of the kernel records)."""
    torch.cuda.synchronize()
    before = sim.launch_count()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        calls()
        torch.cuda.synchronize()
    counted = sim.launch_count() - before
    path = tmp_path / "trace.json"
    prof.export_chrome_trace(str(path))
    with open(path) as f:
        names = [e["name"] for e in json.load(f)["traceEvents"] if e.get("ph") == "X" and e.get("cat") == "kernel"]
    return counted, names


def _check(sim, calls, tmp_path):
    counted, names = _window(sim, calls, tmp_path)
    assert counted > 0
    assert [n for n in names if not LIBRARY_KERNEL.match(n)] == []
    assert len(names) == counted, sorted(set(names))
    return counted


def _steps(sim, n, staged=False):
    def calls():
        for _ in range(n):
            sim.step_staged() if staged else sim.step()
    return calls


def _all_stages(sim):
    s = sim.scene
    sim.enable_contact_events(1 << 14)
    flags = np.zeros(s.n_colliders, np.uint8)
    flags[1::25] = 1
    sim.upload_sensors(flags)
    sim.upload_kinematic_bodies(np.array([(2, (0.0, 0.5, 0.0), (0.0, 0.0, 0.0), 0)], scenes.KINEMATIC))
    f = scenes.default_body_forces(np.arange(3, s.n_bodies, 5))
    f["gravity_scale"] = 0.5
    sim.set_body_forces(f)
    rows = np.zeros(40, nudge_b200.ROW)
    rows["a"] = 3 + 2 * np.arange(40); rows["lin_a"][:, 1] = 1.0; rows["lo"] = -1.0; rows["hi"] = 1.0
    sim.upload_constraint_rows(rows)


def test_parity_staged_calls_on_the_legacy_stream(tmp_path):
    sim = nudge_b200.Sim(_scene())
    sim.step_staged()
    _check(sim, _steps(sim, 3, staged=True), tmp_path)


def test_parity_step_graph_replay(tmp_path):
    sim = nudge_b200.Sim(_scene(), stream=side_stream())
    sim.step(); sim.step()
    assert sim.debug_scalar("graph_active")
    assert _check(sim, _steps(sim, 3), tmp_path) == 3 * 61


@pytest.mark.parametrize("staged", [False, True])
def test_throughput_step(tmp_path, staged):
    sim = nudge_b200.Sim(_scene())
    sim.set_solver_mode("throughput")
    sim.step()
    _check(sim, _steps(sim, 2, staged), tmp_path)


@pytest.mark.parametrize("graph", [False, True])
def test_step_with_every_optional_stage(tmp_path, graph):
    sim = nudge_b200.Sim(_scene(), stream=side_stream() if graph else 0)
    _all_stages(sim)
    sim.step(); sim.step()
    _check(sim, _steps(sim, 2), tmp_path)
    _check(sim, _steps(sim, 1, staged=True), tmp_path)


def test_editing_calls(tmp_path):
    s = _scene()
    sim = nudge_b200.Sim(s, stream=side_stream(), max_bodies=s.n_bodies + 16, max_boxes=s.n_boxes + 16)
    sim.step()
    state = tmp_path / "state.bin"
    sim.save_state(str(state))
    snap = nudge_b200.Snapshot(sim)
    B = s.n_bodies
    impulses = np.zeros(8, scenes.BODY_IMPULSE)
    impulses["body"] = 10 + np.arange(8); impulses["impulse"][:, 1] = 0.25   # not the kinematic body 1

    def calls():
        sim.upload_kinematic_bodies(np.array([(1, (0.0, 0.5, 0.0), (0.0, 0.0, 0.0), 0)], scenes.KINEMATIC))
        sim.apply_body_impulses(impulses)
        sim.apply_radial_impulse((0.0, 0.0, 0.0), 4.0, 2.0)
        sim.set_body_forces(scenes.default_body_forces([B - 1, B - 2]))
        sim.snapshot(into=snap)
        sim.add_bodies(scenes.fragment([(30.0, 2.0, 0.0), (32.0, 2.0, 0.0)], "box", first_tag=1 << 20))
        sim.remove_bodies([3, B + 1])
        sim.restore(snap)
        sim.step()
        sim.load_state(str(state))
        sim.step()

    _check(sim, calls, tmp_path)
