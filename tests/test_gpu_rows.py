"""User constraint rows on the device (nb_upload_constraint_rows, SURVEY.md section 8 f1: the hook of example/main.cpp:316) against the
sequential host loop an application would write there (oracle/rows_ref.py): alone, among the contacts of a pile sweep by sweep in both
solver modes, and at the edges of the row set; and a hanging chain of ball joints as a physical check."""
import numpy as np
import pytest
import nudge_b200
from nudge_b200 import scenes
from oracle import rows_ref, jacobi_ref as J
from tests.parity_util import rows_by_contact, sync_oracle_from_gpu
from tests.test_gpu_throughput import TOL, _rows as _split_rows, _vel, assert_velocities_close

pytestmark = pytest.mark.gpu
ROWS_TOL = 2e-5     # float32 kernel against the float64 loop, relative to the velocity (impulse) scale


def _quat_rotate(q, v):
    x, y, z, w = q
    t = 2.0 * np.cross(q[:3], v)
    return v + w * t + np.cross(q[:3], t)


def _quat_unrotate(q, v):
    return _quat_rotate(np.array([-q[0], -q[1], -q[2], q[3]]), v)


def _random_rows(rng, m, a, b):
    """Generic rows on the given bodies: random Jacobians and biases, about a third unilateral (lo = 0), a fifth bounded above, half
    soft, warm-started from nonzero impulses."""
    rows = np.zeros(m, nudge_b200.ROW)
    rows["a"], rows["b"] = a, b
    for k in ("lin_a", "ang_a", "lin_b", "ang_b"):
        rows[k] = rng.normal(size=(m, 3))
    rows["bias"] = rng.normal(size=m) * 0.3
    rows["lo"] = np.where(rng.random(m) < 0.3, 0.0, -np.inf); rows["hi"] = np.where(rng.random(m) < 0.2, 0.5, np.inf)
    rows["impulse"] = np.where(rows["lo"] == 0.0, 0.1, rng.normal(size=m) * 0.1); rows["softness"] = np.where(rng.random(m) < 0.5, 0.01, 0.0)
    return rows


def _free_bodies(n, iterations, seed=3):
    """n bodies far apart and far above the ground, randomly rotated and moving, no gravity: a step has no contacts."""
    s = scenes.demo_scene(n, 0, iterations=iterations, spread=200.0, height=10.0, seed=seed)
    s.transforms["position"][1:, 1] += 500.0
    rng = np.random.default_rng(1)
    s.transforms["rotation"][1:] = scenes._random_unit_quaternions(rng, n)
    s.momentum["velocity"][1:] = rng.normal(size=(n, 3)); s.momentum["angular_velocity"][1:] = rng.normal(size=(n, 3))
    s.gravity = np.float32(0.0); s.damping = np.float32(0.0)
    return s, rng


def _world_inertia(g):
    g.download_bodies()
    return rows_ref.world_inverse_inertia(g.transforms["rotation"], g.scene.properties["inertia_inverse"]), g.scene.properties["mass_inverse"].astype(np.float64)


def _assert_rows_close(g, lin, ang, want, what):
    g.download_bodies()
    scale = max(1.0, np.abs(lin).max(), np.abs(ang).max())
    assert np.abs(g.momentum["velocity"] - lin).max() < ROWS_TOL * scale, what
    assert np.abs(g.momentum["angular_velocity"] - ang).max() < ROWS_TOL * scale, what
    got = g.download_constraint_rows(len(want))
    assert np.abs(got["impulse"] - want["impulse"]).max() < ROWS_TOL * max(1.0, np.abs(want["impulse"]).max()), what
    return got


def ball_joint_rows(xf, a, b, anchor_a, anchor_b, dt, beta=0.2):
    """Three rows holding the world-space anchors of bodies a and b together (b = 0: a point fixed in the world)."""
    pa, qa = xf["position"][a].astype(np.float64), xf["rotation"][a].astype(np.float64)
    ra = _quat_rotate(qa, np.asarray(anchor_a, np.float64))
    if b:
        pb, qb = xf["position"][b].astype(np.float64), xf["rotation"][b].astype(np.float64)
        rb = _quat_rotate(qb, np.asarray(anchor_b, np.float64)); wb = pb + rb
    else:
        rb = np.zeros(3); wb = np.asarray(anchor_b, np.float64)
    err = (pa + ra) - wb
    rows = np.zeros(3, nudge_b200.ROW)
    for k in range(3):
        e = np.zeros(3); e[k] = 1.0
        rows[k]["a"], rows[k]["b"] = a, b
        rows[k]["lin_a"] = e; rows[k]["ang_a"] = np.cross(ra, e)
        rows[k]["lin_b"] = -e; rows[k]["ang_b"] = -np.cross(rb, e)
        rows[k]["bias"] = beta / dt * err[k]
        rows[k]["lo"], rows[k]["hi"] = -np.inf, np.inf
    return rows


def test_rows_equal_the_sequential_host_loop():
    """No contacts (bodies far apart, far above the ground): the solver stage is the user rows alone, applied after each of the 5 sweeps."""
    _rows_alone_equal_the_sequential_host_loop("parity")


def test_rows_equal_the_sequential_host_loop_in_throughput_mode():
    """The same in throughput mode: the rows run after every Jacobi pass (which has no contacts to solve here)."""
    _rows_alone_equal_the_sequential_host_loop("throughput")


def _rows_alone_equal_the_sequential_host_loop(mode):
    n = 40
    s, rng = _free_bodies(n, 5)
    g = nudge_b200.Sim(s)
    g.set_solver_mode(mode)
    m = 150
    rows = np.zeros(m, nudge_b200.ROW)
    rows["a"] = rng.integers(0, n + 1, m); rows["b"] = rng.integers(0, n + 1, m)
    same = rows["a"] == rows["b"]; rows["b"][same] = (rows["a"][same] % n) + 1
    for k in ("lin_a", "ang_a", "lin_b", "ang_b"):
        rows[k] = rng.normal(size=(m, 3))
    rows["bias"] = rng.normal(size=m) * 0.3
    rows["lo"] = np.where(rng.random(m) < 0.3, 0.0, -np.inf); rows["hi"] = np.where(rng.random(m) < 0.2, 0.5, np.inf)
    rows["impulse"] = np.where(rows["lo"] == 0.0, 0.1, rng.normal(size=m) * 0.1); rows["softness"] = np.where(rng.random(m) < 0.5, 0.01, 0.0)
    g.upload_constraint_rows(rows)
    want = rows.copy()
    lin, ang = s.momentum["velocity"].astype(np.float64), s.momentum["angular_velocity"].astype(np.float64)
    I = rows_ref.world_inverse_inertia(s.transforms["rotation"], s.properties["inertia_inverse"])
    minv = s.properties["mass_inverse"].astype(np.float64)
    rows_ref.apply_rows(want, lin, ang, minv, I, warm=True)
    for _ in range(5):
        rows_ref.apply_rows(want, lin, ang, minv, I)
    g.collide(); g.apply_gravity_damping(); g.read_cached_impulses(); g.setup_contact_constraints(); g.apply_impulses(5)
    assert g.counts().contacts == 0
    g.download_bodies()
    got = g.download_constraint_rows(m)
    scale = max(1.0, np.abs(lin).max(), np.abs(ang).max())
    assert np.abs(g.momentum["velocity"] - lin).max() < 2e-5 * scale and np.abs(g.momentum["angular_velocity"] - ang).max() < 2e-5 * scale
    assert np.abs(got["impulse"] - want["impulse"]).max() < 2e-5 * max(1.0, np.abs(want["impulse"]).max())
    # nb_step (graph replay on a created stream) takes the same path
    import torch
    side = torch.cuda.Stream()
    h = nudge_b200.Sim(s, stream=side.cuda_stream)
    h.set_solver_mode(mode)
    h.upload_constraint_rows(rows)
    h.step(); g.update_cached_impulses(); g.write_cached_impulses(); g.advance()
    h.download_bodies(); g.download_bodies()
    assert h.momentum.tobytes() == g.momentum.tobytes() and h.transforms.tobytes() == g.transforms.tobytes()
    g.upload_constraint_rows(np.zeros(0, nudge_b200.ROW))        # removing the rows restores the plain step
    g.step_staged()


def test_hanging_chain_of_ball_joints_stays_connected_among_contacts():
    """A 10-link chain hung from the world by ball joints swings into a pile of loose boxes: the anchors stay together (joint error
    bounded) while ordinary contacts are solved around it; the joint bodies are connected for the island pass (example/main.cpp:285)."""
    links = 10
    s = scenes.demo_scene(links + 60, 0, iterations=12, spread=3.0, height=6.0, seed=5)
    s.box_data["size"][1:links + 1] = (0.2, 0.5, 0.2)
    s.properties[1:links + 1] = scenes._box_props(s.box_data["size"][1:links + 1])
    top = np.array([6.0, 8.0, 0.0])
    for k in range(links):                                    # laid out horizontally: it will swing down
        s.transforms["position"][1 + k] = top + np.array([0.5 + 1.0 * k, 0.0, 0.0])
        s.transforms["rotation"][1 + k] = (0.0, 0.0, np.sin(np.pi / 4), np.cos(np.pi / 4))   # long axis along x
    s.connections = np.zeros(links - 1, scenes.PAIR32); s.connections["a"] = 1 + np.arange(links - 1); s.connections["b"] = 2 + np.arange(links - 1)
    g = nudge_b200.Sim(s)
    dt = float(s.time_step)
    worst = 0.0
    for step in range(240):
        g.download_bodies()
        rows = [ball_joint_rows(g.transforms, 1, 0, (0.0, 0.5, 0.0), top, dt)]
        for k in range(1, links):
            rows.append(ball_joint_rows(g.transforms, 1 + k, k, (0.0, 0.5, 0.0), (0.0, -0.5, 0.0), dt))
        g.upload_constraint_rows(np.concatenate(rows))
        g.step_staged()
        if step > 20:
            g.download_bodies()
            for k in range(1, links):
                wa = g.transforms["position"][1 + k] + _quat_rotate(g.transforms["rotation"][1 + k].astype(np.float64), np.array([0.0, 0.5, 0.0]))
                wb = g.transforms["position"][k] + _quat_rotate(g.transforms["rotation"][k].astype(np.float64), np.array([0.0, -0.5, 0.0]))
                worst = max(worst, float(np.linalg.norm(wa - wb)))
    assert worst < 0.08, worst
    assert np.isfinite(g.transforms["position"]).all() and g.counts().overflow == 0
    end = g.transforms["position"][links]
    assert end[1] < top[1] - 0.5 * links                     # the chain hangs below its support now


# ---------------- rows among contacts ----------------

def _pile():
    """A small settled pile: 300 bodies, 300 contacts after 60 steps."""
    return scenes.demo_scene(150, 150, iterations=6, spread=3.0, height=12.0)


def _rows_among_contacts(g, seed=7):
    """Rows on a pile the GPU simulation g has just stepped: ball joints (anchor at the midpoint, so the error starts at zero) between
    40 pairs of bodies in contact, generic rows with the world on side a or b and between two bodies, and 40 rows on one body of the
    pile (40 levels).  Interleaved, so that rows of different kinds share levels."""
    rng = np.random.default_rng(seed)
    g.download_bodies(); g.download_contacts()
    xf, dt = g.transforms, float(g.scene.time_step)
    ab = g.contact_bodies[:g.contacts.count]
    pairs = np.unique(np.stack([ab["a"], ab["b"]], 1).astype(np.int64), axis=0)
    pairs = pairs[(pairs[:, 0] != 0) & (pairs[:, 1] != 0)]
    assert len(pairs) >= 40
    joints = []
    for a, b in pairs[rng.choice(len(pairs), 40, replace=False)]:
        pa, pb = xf["position"][a].astype(np.float64), xf["position"][b].astype(np.float64)
        mid = 0.5 * (pa + pb)
        joints.append(ball_joint_rows(xf, a, b, _quat_unrotate(xf["rotation"][a].astype(np.float64), mid - pa),
                                      _quat_unrotate(xf["rotation"][b].astype(np.float64), mid - pb), dt))
    B = g.scene.n_bodies
    m = 150
    a, b = rng.integers(1, B, m), rng.integers(1, B, m)
    side = rng.random(m)
    b[side < 0.3] = 0; a[(side >= 0.3) & (side < 0.6)] = 0
    b[(a == b) & (a != 0)] = 0
    hub = int(pairs[0][0])
    other = rng.integers(1, B, 40); other[other == hub] = 0; other[::4] = 0
    flip = rng.random(40) < 0.5
    hub_rows = _random_rows(rng, 40, np.where(flip, other, hub), np.where(flip, hub, other))
    rows = np.concatenate(joints + [_random_rows(rng, m, a, b), hub_rows])
    rows = rows[rng.permutation(len(rows))]
    assert ((rows["a"] == hub) | (rows["b"] == hub)).sum() >= 30
    assert not ((rows["a"] == rows["b"]) & (rows["a"] != 0)).any()
    return rows


def test_rows_between_contact_sweeps_equal_the_oracle_then_the_host_loop():
    """Parity mode, stage by stage: after setup the GPU equals the oracle's warm start followed by the rows' warm start; before every
    sweep the oracle and the row copy take the GPU's momentum and row impulses, then run one contact sweep and one pass of the rows.
    The contact states and the momentum's unused lanes (inverse mass, sweep token) are a function of shared state: bit for bit."""
    from oracle import pyoracle
    s = _pile()
    o = pyoracle.OracleSim(s)
    g = nudge_b200.Sim(s, contact_capacity=o.cap, debug=True)
    assert g.lut_model_exact()
    for _ in range(60):
        g.step()
    rows = _rows_among_contacts(g)
    g.upload_constraint_rows(rows)
    want = rows.copy()
    sync_oracle_from_gpu(o, g)
    o.collide(); g.collide()
    assert o.contacts.count == g.counts().contacts > 200
    n = o.contacts.count
    o.apply_gravity_damping(); g.apply_gravity_damping()
    o.read_cached_impulses(); g.read_cached_impulses()
    o.setup_contact_constraints(); g.setup_contact_constraints()
    I, minv = _world_inertia(g)

    def check(what):
        gk = g.constraints_view()
        ok = rows_by_contact(o.constraints_view(), n)
        assert np.array_equal(ok["states"][gk["contact"].astype(np.int64)].view(np.uint32), gk["states"].view(np.uint32)), what + ": contact states"
        g.download_bodies()
        for lane in ("unused0", "unused1"):
            assert o.momentum[lane].tobytes() == g.momentum[lane].tobytes(), what + ": " + lane
        lin, ang = o.momentum["velocity"].astype(np.float64), o.momentum["angular_velocity"].astype(np.float64)
        rows_ref.apply_rows(want, lin, ang, minv, I, warm=what == "warm start")
        return _assert_rows_close(g, lin, ang, want, what)

    got = check("warm start")
    for sweep in range(int(s.iterations)):
        o.momentum[:] = g.momentum; want["impulse"] = got["impulse"]
        o.apply_impulses(); g.apply_impulses(1)
        got = check("sweep %d" % sweep)
    assert g.counts().overflow == 0


def test_rows_between_throughput_sweeps_equal_the_restatement_then_the_host_loop():
    """The same loop in throughput mode: a Jacobi pass (oracle/jacobi_ref.py) in place of the oracle's sweep, within its tolerance."""
    s = _pile()
    g = nudge_b200.Sim(s, debug=True)
    for _ in range(60):
        g.step()
    rows = _rows_among_contacts(g)
    g.set_solver_mode("throughput")
    g.upload_constraint_rows(rows)
    want = rows.copy()
    g.collide(); g.apply_gravity_damping(); g.read_cached_impulses()
    lin, ang = _vel(g)
    g.setup_contact_constraints()
    n = g.counts().contacts
    assert n > 200
    P, st, ct, a, b = _split_rows(g, n)
    cnt = g.debug("body_contacts", np.uint32).astype(np.int64)[:s.n_bodies]
    I, minv = _world_inertia(g)
    imp = g.impulses_view()["data"]["impulse"][ct]
    for sweep in range(-1, int(s.iterations)):
        if sweep >= 0:
            want["impulse"] = g.download_constraint_rows(len(rows))["impulse"]
            g.apply_impulses(1)
        r = J.jacobi_pass(P, st, a, b, lin, ang, warm=sweep < 0, impulses=imp, abs_sums=True)
        lin_w, ang_w = r[0].copy(), r[1].copy()
        rows_ref.apply_rows(want, lin_w, ang_w, minv, I, warm=sweep < 0)
        what = "warm start" if sweep < 0 else "sweep %d" % sweep
        lin, ang = _vel(g)
        assert_velocities_close(lin, ang, (lin_w, ang_w) + r[2:], cnt, what)
        _, st, _, _, _ = _split_rows(g, n)
        assert np.abs(st - r[2]).max() < TOL * max(1.0, np.abs(r[2]).max()), what
        got = g.download_constraint_rows(len(rows))
        assert np.abs(got["impulse"] - want["impulse"]).max() < TOL * max(1.0, np.abs(want["impulse"]).max()), what
    assert g.counts().overflow == 0


def test_step_graph_with_rows_and_contacts_equals_the_staged_calls():
    """nb_step (graph replay on a created stream) against the seven stage calls, with rows among contacts: bit for bit, 20 steps."""
    import torch
    s = _pile()
    side = torch.cuda.Stream()
    g, h = nudge_b200.Sim(s), nudge_b200.Sim(s, stream=side.cuda_stream)
    for _ in range(60):
        g.step_staged(); h.step()
    rows = _rows_among_contacts(g)
    g.upload_constraint_rows(rows); h.upload_constraint_rows(rows)
    for step in range(20):
        g.step_staged(); h.step()
        g.download_bodies(); h.download_bodies()
        assert h.momentum.tobytes() == g.momentum.tobytes() and h.transforms.tobytes() == g.transforms.tobytes(), "step %d" % step
    assert g.counts().contacts > 100
    assert g.download_constraint_rows(len(rows)).tobytes() == h.download_constraint_rows(len(rows)).tobytes()


# ---------------- edges of the row set ----------------

def _assert_next_step_equals_one_without_rows(g, s):
    """g's rows were refused: its next step must be byte for byte that of a simulation that never had rows."""
    r = nudge_b200.Sim(s)
    assert g.download_constraint_rows(0).size == 0
    g.step_staged(); r.step_staged()
    g.download_bodies(); r.download_bodies()
    assert g.momentum.tobytes() == r.momentum.tobytes() and g.transforms.tobytes() == r.transforms.tobytes()


def test_a_chain_of_4096_levels_is_accepted_and_4097_are_refused():
    s, rng = _free_bodies(40, 2)
    other = rng.integers(2, 41, 4096); other[::3] = 0
    flip = rng.random(4096) < 0.5
    rows = _random_rows(rng, 4096, np.where(flip, other, 1), np.where(flip, 1, other))     # every row on body 1: 4096 levels
    g = nudge_b200.Sim(s)
    g.upload_constraint_rows(rows)
    want = rows.copy()
    I, minv = _world_inertia(g)
    lin, ang = s.momentum["velocity"].astype(np.float64), s.momentum["angular_velocity"].astype(np.float64)
    rows_ref.apply_rows(want, lin, ang, minv, I, warm=True)
    for _ in range(int(s.iterations)):
        rows_ref.apply_rows(want, lin, ang, minv, I)
    g.collide(); g.apply_gravity_damping(); g.read_cached_impulses(); g.setup_contact_constraints(); g.apply_impulses(int(s.iterations))
    assert g.counts().contacts == 0
    _assert_rows_close(g, lin, ang, want, "4096 levels")
    # one more row on body 1: refused, and the set it replaces is gone
    g = nudge_b200.Sim(s)
    g.upload_constraint_rows(rows)
    with pytest.raises(nudge_b200.NudgeError, match=r"4096 levels.*\(-2\)"):
        g.upload_constraint_rows(np.concatenate([rows, rows[:1]]))
    _assert_next_step_equals_one_without_rows(g, s)


def test_rows_on_one_body_twice_or_beyond_max_bodies_are_refused():
    """a == b != 0 (the effective mass would need cross terms; put the whole Jacobian on a, b = 0) and a body >= max_bodies are
    argument errors that remove the set; a == b == 0 is legal, computes its impulse and touches no body."""
    s, rng = _free_bodies(40, 3)
    good = _random_rows(rng, 20, rng.integers(1, 21, 20), rng.integers(21, 41, 20))
    beyond = s.n_bodies                         # the first index beyond max_bodies (= the scene's body count here)
    for bad_a, bad_b, text in ((5, 5, "same body"), (beyond, 0, "max_bodies"), (0, beyond, "max_bodies"), (7, 1 << 20, "max_bodies")):
        g = nudge_b200.Sim(s)
        g.upload_constraint_rows(good)
        rows = good.copy()
        rows[11]["a"], rows[11]["b"] = bad_a, bad_b
        with pytest.raises(nudge_b200.NudgeError, match=text + r".*\(-3\)"):
            g.upload_constraint_rows(rows)
        _assert_next_step_equals_one_without_rows(g, s)
    # both sides on the world: accepted; the impulse follows the host loop, no velocity changes
    g, r = nudge_b200.Sim(s), nudge_b200.Sim(s)
    rows = good.copy(); rows[11]["a"] = rows[11]["b"] = 0
    g.upload_constraint_rows(rows[11:12])
    g.step_staged(); r.step_staged()
    g.download_bodies(); r.download_bodies()
    assert g.momentum.tobytes() == r.momentum.tobytes()
    want = rows[11:12].copy()
    z = np.zeros((s.n_bodies, 3))
    I, minv = _world_inertia(g)
    rows_ref.apply_rows(want, z, z.copy(), minv, I, warm=True)
    for _ in range(int(s.iterations)):
        rows_ref.apply_rows(want, z, z.copy(), minv, I)
    assert abs(float(g.download_constraint_rows(1)["impulse"][0]) - float(want["impulse"][0])) < ROWS_TOL * max(1.0, abs(float(want["impulse"][0])))


def test_download_with_a_different_row_count_is_refused():
    s, rng = _free_bodies(40, 2)
    g = nudge_b200.Sim(s)
    rows = _random_rows(rng, 30, rng.integers(1, 21, 30), rng.integers(21, 41, 30))
    g.upload_constraint_rows(rows)
    for n in (29, 31, 0):
        with pytest.raises(nudge_b200.NudgeError, match=r"differs.*\(-3\)"):
            g.download_constraint_rows(n)
    assert g.download_constraint_rows(30).tobytes() == rows.tobytes()


def _disjoint_rows_pass(rows, lin, ang, minv, I, warm=False):
    """rows_ref.apply_rows, vectorised: only valid for rows that touch pairwise disjoint bodies (then the order of the loop is free)."""
    a, b = rows["a"].astype(np.int64), rows["b"].astype(np.int64)
    la, aa, lb, ab = (rows[k].astype(np.float64) for k in ("lin_a", "ang_a", "lin_b", "ang_b"))
    ma, mb = np.where(a != 0, minv[a], 0.0), np.where(b != 0, minv[b], 0.0)
    ia = np.where((a != 0)[:, None], np.einsum("nij,nj->ni", I[a], aa), 0.0)
    ib = np.where((b != 0)[:, None], np.einsum("nij,nj->ni", I[b], ab), 0.0)
    imp = rows["impulse"].astype(np.float64)
    if warm:
        delta = imp
    else:
        dot = lambda x, y: (x * y).sum(1)
        soft = rows["softness"].astype(np.float64)
        k = ma * dot(la, la) + dot(aa, ia) + mb * dot(lb, lb) + dot(ab, ib) + soft
        jv = dot(la, lin[a]) + dot(aa, ang[a]) + dot(lb, lin[b]) + dot(ab, ang[b])
        eff = np.where(k > 0, 1.0 / np.where(k > 0, k, 1.0), 0.0)
        nxt = np.minimum(np.maximum(imp - eff * (jv + rows["bias"] + soft * imp), rows["lo"]), rows["hi"])
        delta = nxt - imp
        rows["impulse"] = nxt
    sa, sb = a != 0, b != 0
    lin[a[sa]] += (ma[:, None] * la * delta[:, None])[sa]; ang[a[sa]] += (ia * delta[:, None])[sa]
    lin[b[sb]] += (mb[:, None] * lb * delta[:, None])[sb]; ang[b[sb]] += (ib * delta[:, None])[sb]


def test_one_level_wider_than_the_grid():
    """More rows in one level than SMs x 8 blocks x 256 threads: k_user_rows walks them with its grid-stride loop."""
    import torch
    width = torch.cuda.get_device_properties(0).multi_processor_count * 8 * 256
    m = width + 1000
    third = m // 3
    nb = 2 * third + (m - third)                 # pairs, then rows on one body against the world (a = 0 or b = 0)
    rng = np.random.default_rng(11)
    side = int(np.ceil(nb ** (1 / 3)))
    k = np.arange(nb)
    pos = np.stack([(k % side) * 3.0, 500.0 + (k // (side * side)) * 3.0, ((k // side) % side) * 3.0], 1).astype(np.float32)
    s = scenes._assemble("row_level", np.zeros((0, 3), np.float32), np.zeros((0, 3), np.float32), None, np.full(nb, 0.5, np.float32), pos)
    s.transforms["rotation"][1:] = scenes._random_unit_quaternions(rng, nb)
    s.momentum["velocity"][1:] = rng.normal(size=(nb, 3)); s.momentum["angular_velocity"][1:] = rng.normal(size=(nb, 3))
    s.gravity = np.float32(0.0); s.damping = np.float32(0.0); s.iterations = 2
    body = 1 + rng.permutation(nb)
    a = np.concatenate([body[:third], body[2 * third:2 * third + (m - third) // 2], np.zeros(m - third - (m - third) // 2, np.int64)])
    b = np.concatenate([body[third:2 * third], np.zeros((m - third) // 2, np.int64), body[2 * third + (m - third) // 2:]])
    rows = _random_rows(rng, m, a, b)
    used = np.concatenate([a[a != 0], b[b != 0]])
    assert m > width and len(np.unique(used)) == len(used), "one level: pairwise disjoint rows"
    g = nudge_b200.Sim(s, contact_capacity=4096)
    g.upload_constraint_rows(rows)
    I, minv = _world_inertia(g)
    lin, ang = s.momentum["velocity"].astype(np.float64), s.momentum["angular_velocity"].astype(np.float64)
    # the vectorised pass is the host loop on disjoint rows: checked on a sample of every kind first
    sub, l2, a2 = rows[::97].copy(), lin.copy(), ang.copy()
    rows_ref.apply_rows(sub, l2, a2, minv, I)
    sub2, l3, a3 = rows[::97].copy(), lin.copy(), ang.copy()
    _disjoint_rows_pass(sub2, l3, a3, minv, I)
    assert np.abs(l2 - l3).max() < 1e-9 and np.abs(a2 - a3).max() < 1e-9 and np.abs(sub["impulse"] - sub2["impulse"]).max() < 1e-9
    want = rows.copy()
    _disjoint_rows_pass(want, lin, ang, minv, I, warm=True)
    for _ in range(int(s.iterations)):
        _disjoint_rows_pass(want, lin, ang, minv, I)
    g.collide(); g.apply_gravity_damping(); g.read_cached_impulses(); g.setup_contact_constraints(); g.apply_impulses(int(s.iterations))
    assert g.counts().contacts == 0
    got = _assert_rows_close(g, lin, ang, want, "one level of %d rows" % m)
    assert (got["impulse"] != rows["impulse"]).mean() > 0.9          # the rows beyond the first grid's worth ran too
