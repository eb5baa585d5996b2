"""Throughput-mode solver (mass-splitting Jacobi, nudge_b200/csrc/nb_jacobi.cuh) on the GPU, through the C ABI.

It is NOT bit-comparable with the reference (different iteration, float atomics): the split rows and every pass are compared with
the CPU restatement oracle/jacobi_ref.py within a stated tolerance (1e-4 of the velocity scale; the restatement is float64 with exact
1/x and 1/sqrt, the kernel float32 with the GPU's reciprocal/rsqrt; plus, per body, the rounding of a float32 sum in free order),
and the physics is compared with parity mode through invariants."""
import numpy as np
import pytest
import nudge_b200
from nudge_b200 import scenes
from oracle import jacobi_ref as J

pytestmark = pytest.mark.gpu
TOL = 1e-4
TWO_STAGE_BODIES = 600000     # above this body count k_jacobi_sweep runs its two-stage ring (jacobi_stages() in nb_api.cu)


def _rows(g, n):
    stride = g.debug_scalar("row_stride")
    P = g.debug("row_planes_all", np.float32).reshape(41, stride)
    st = g.debug("row_states", np.float32).reshape(3, stride)
    contact = g.debug("row_contact", np.uint32)
    used = np.nonzero(contact != 0xffffffff)[0]
    assert len(used) == n
    return P[:, used], st[:, used], contact[used].astype(np.int64), g.debug("row_a", np.uint32)[used].astype(np.int64), g.debug("row_b", np.uint32)[used].astype(np.int64)


def _vel(g):
    g.download_bodies()
    return g.momentum["velocity"].astype(np.float64), g.momentum["angular_velocity"].astype(np.float64)


def assert_velocities_close(lin, ang, want, cnt, what):
    """want = jacobi_pass(..., abs_sums=True).  Per body and component: |got - want| < TOL * scale + 2 cnt 2^-24 sum|delta|, the second
    term being the rounding of the kernel's float32 sums of cnt contact changes in free order (warp shuffles, then atomics)."""
    lin_w, ang_w, _, alin, aang = want
    scale = max(1.0, np.abs(lin_w).max(), np.abs(ang_w).max())
    slack = 2.0 * cnt[:, None] * 2.0 ** -24
    for name, got, ref, asum in (("linear", lin, lin_w, alin), ("angular", ang, ang_w, aang)):
        err, bound = np.abs(got - ref), TOL * scale + slack * asum
        bad = np.argwhere(err >= bound)
        assert not len(bad), "%s %s velocity: %d components out of bound, first body %d (%d contacts): error %g, bound %g" % (
            what, name, len(bad), bad[0][0], cnt[bad[0][0]], err[tuple(bad[0])], bound[tuple(bad[0])])


def _ring_scene():
    """More than 600,000 bodies, so the two-stage ring runs: a running-bond wall of 32,768 bricks overlapping by 1e-3 (in contact from
    the first step: 535,581 contacts after two steps, 2,093 tiles) under a sparse lattice of 580,000 small spheres far above it that
    touch nothing during the test."""
    w = scenes.brick_wall(32768, gap=-1e-3)
    nx, ny = 100, 58
    k = np.arange(nx * nx * ny)
    sph = np.stack([(k % nx - nx / 2) * 3.0, 400.0 + (k // (nx * nx)) * 3.0, ((k // nx) % nx - nx / 2) * 3.0], 1).astype(np.float32)
    s = scenes._assemble("ring", w.box_data["size"][1:], w.transforms["position"][1:], None, np.full(len(k), 0.5, np.float32), sph,
                         ground_half=tuple(w.box_data["size"][0]), ground_y=float(w.box_transforms["position"][0][1]))
    s.iterations = w.iterations
    return s


def _hub_scene():
    """scenes.hub_platform(55) with the small boxes moving down onto the platform at 2 m/s.  After one step the platform's velocity
    changes by about 0.48 m/s in the warm start and in the first sweep, the sum of 12,100 contacts; with the boxes at rest it changes
    by under 1e-2, and by nothing after two steps, where a wrong sum would hide inside the tolerance."""
    s = scenes.hub_platform(55)
    s.momentum["velocity"][2:, 1] = -2.0
    return s


# name: (scene, settle steps, contact capacity (None: the default of 24 per body))
CASES = {
    "mixed": (lambda: scenes.demo_scene(400, 400, iterations=8, spread=4.0, height=10.0), 260, None),
    "boxes": (lambda: scenes.box_drop(3000, iterations=8, density_L=30.0), 260, None),
    "ring": (_ring_scene, 2, 1100000),
    "hub": (_hub_scene, 1, None),                                  # 12,100 contacts on one dynamic body: runs of 32 across warps and tiles
    "tiny": (scenes.two_boxes, 2, None),                           # 8 contacts: one partial tile
    "none": (lambda: scenes.two_boxes(pos_b=(0.0, 10.0, 0.0)), 2, None),
}


def _check_premises(case, g, scene, n, a, b, cnt):
    """What each case is there to reach; a scene that stops reaching it fails here instead of silently testing something else."""
    tiles = (n + 255) // 256
    stages, blocks = g.debug_scalar("jacobi_stages"), g.debug_scalar("jacobi_blocks")
    assert stages == (2 if scene.n_bodies > TWO_STAGE_BODIES else 1)
    print("%s: %d bodies, %d contacts, %d tiles, k_jacobi_sweep<*, %d> on %d CTAs" % (case, scene.n_bodies, n, tiles, stages, blocks))
    if case in ("mixed", "boxes"):
        assert n > 500
    elif case == "ring":
        assert stages == 2 and tiles >= 5 * blocks and n % 256, "every CTA must refill both stages and see both mbarrier parities"
        assert max(a.max(), b.max()) <= scene.n_boxes - 1, "the spheres must not touch anything"
    elif case == "hub":
        platform = 1
        assert cnt[platform] == n == np.count_nonzero((a == platform) | (b == platform)) and n >= 12100
    elif case == "tiny":
        assert 0 < n < 256
    else:
        assert n == 0


@pytest.mark.parametrize("case", list(CASES))
def test_split_rows_warm_start_and_sweeps_equal_the_cpu_restatement(case):
    make, settle, capacity = CASES[case]
    scene = make()
    g = nudge_b200.Sim(scene, contact_capacity=capacity, debug=True)
    for _ in range(settle):
        g.step_staged()
    g.collide(); g.apply_gravity_damping(); g.read_cached_impulses()
    g.download_bodies(); m0 = g.momentum.copy()
    n = g.counts().contacts
    # the same contact set through the exact-order setup (rows pinned bit-for-bit against the reference in test_gpu_parity.py)
    g.setup_contact_constraints()
    Pp, _, cp, ap, bp = _rows(g, n)
    order = np.argsort(cp)
    Pp, ap, bp = Pp[:, order], ap[order], bp[order]                 # keyed by contact index
    g.momentum[:] = m0; g.upload_bodies()
    g.set_solver_mode("throughput")
    assert g.solver_mode() == "throughput"
    g.setup_contact_constraints()                                   # split rows + Jacobi warm start
    Pt, st, ct, a, b = _rows(g, n)
    assert np.array_equal(ct, g.debug("sorted", np.uint32).astype(np.int64)), "throughput slots are the tag order"
    assert np.array_equal(a, ap[ct]) and np.array_equal(b, bp[ct])
    cnt = g.debug("body_contacts", np.uint32).astype(np.int64)[:scene.n_bodies]
    want_cnt = np.bincount(np.concatenate([a, b]), minlength=scene.n_bodies); want_cnt[0] = 0
    assert np.array_equal(cnt, want_cnt)
    _check_premises(case, g, scene, n, a, b, cnt)
    if n == 0:       # no tiles: the warm start and the sweeps must leave every velocity as it was
        g.apply_impulses(3)
        g.download_bodies()
        assert g.momentum.tobytes() == m0.tobytes()
        return
    split = {"NVTNI", "BIAS", "FC_X", "FC_Y", "FC_Z"}
    for k, name in enumerate(J.PLANES):
        if name not in split:
            assert np.array_equal(Pt[k].view(np.uint32), Pp[k][ct].view(np.uint32)), name     # everything else is the reference's row, bit for bit
    t = J.split_terms(Pp[:, ct], a, b, cnt)
    for name in split:
        got = Pt[J.IX[name]].astype(np.float64)
        assert np.abs(got - t[name]).max() <= 2e-5 * np.abs(t[name]).max(), name
    # warm start, then three sweeps, each against the restatement started from the GPU's own previous state
    lin0, ang0 = m0["velocity"].astype(np.float64), m0["angular_velocity"].astype(np.float64)
    imp = g.impulses_view()["data"]["impulse"][ct]
    want = J.jacobi_pass(Pt, st, a, b, lin0, ang0, warm=True, impulses=imp, abs_sums=True)
    lin, ang = _vel(g)
    if case == "hub":
        assert np.abs(want[0][1] - lin0[1]).max() > 1000 * TOL, "the platform's warm start must be far larger than the tolerance"
    assert_velocities_close(lin, ang, want, cnt, "warm start")
    assert np.abs(st - want[2]).max() < TOL * max(1.0, np.abs(want[2]).max())
    for sweep in range(3):
        want = J.jacobi_pass(Pt, st, a, b, lin, ang, abs_sums=True)
        g.apply_impulses(1)
        lin, ang = _vel(g)
        _, st, _, _, _ = _rows(g, n)
        assert_velocities_close(lin, ang, want, cnt, "sweep %d" % sweep)
        assert np.abs(st - want[2]).max() < TOL * max(1.0, np.abs(want[2]).max()), "sweep %d" % sweep
    assert g.counts().overflow == 0


def _pile_stats(g):
    g.collide(); g.download_contacts(); g.download_bodies()
    n = g.contacts.count
    pen = g.contact_data["penetration"][:n]
    v = g.momentum["velocity"][1:]
    mass = 1.0 / g.properties["mass_inverse"][1:]
    return dict(contacts=n, max_pen=float(pen.max()), mean_pen=float(pen.mean()), ke=float(0.5 * (mass * (v * v).sum(1)).sum()),
                mean_y=float(g.transforms["position"][1:, 1].mean()), min_y=float(g.transforms["position"][1:, 1].min()))


def test_throughput_mode_keeps_a_settled_pile_settled_like_parity_mode():
    """Invariants vs parity mode on a settled 8k pile, 120 further steps each: nothing sinks or explodes, penetration and
    kinetic energy stay in the same range.  nb_step (CUDA graph) drives the throughput run."""
    import torch
    s = scenes.box_drop(8000, iterations=8, density_L=45.0)     # 8 layers over a wide footprint: at rest after ~400 steps
    side = torch.cuda.Stream()
    a = nudge_b200.Sim(s, stream=side.cuda_stream)
    for _ in range(700):
        a.step()
    a.download_bodies(); a.download_cache()
    b = nudge_b200.Sim(s, stream=side.cuda_stream)
    for name in ("transforms", "momentum", "idle"):
        getattr(b, name)[:] = getattr(a, name)
    nc = a.cache.count
    b.cache_tags[:nc] = a.cache_tags[:nc]; b.cache_features[:nc] = a.cache_features[:nc]; b.cache_data[:nc] = a.cache_data[:nc]; b.cache.count = nc
    b.upload_bodies(); b.upload_cache()
    b.set_solver_mode("throughput")
    for _ in range(120):
        a.step(); b.step()
    sa, sb = _pile_stats(a), _pile_stats(b)
    print("parity    ", sa); print("throughput", sb)
    assert b.counts().overflow == 0
    assert np.isfinite(b.transforms["position"]).all()
    assert sb["min_y"] > -1.0                                            # nothing fell through the ground (top at y = 0)
    assert abs(sb["mean_y"] - sa["mean_y"]) < 0.05 * max(1.0, abs(sa["mean_y"]))
    # Jacobi with 8 sweeps is softer than Gauss-Seidel with 8 sweeps: the pile rests deeper (more penetration, hence more contacts), but
    # it rests.  Measured on the falling 8k column of the first version of this test: mean penetration 0.053 vs 0.014, contacts +20 %.
    assert sb["max_pen"] < 4.0 * sa["max_pen"] + 0.1 and sb["mean_pen"] < 6.0 * sa["mean_pen"] + 0.02
    assert sb["ke"] < 10.0 * sa["ke"] + 50.0                              # still at rest (the falling pile had > 1e6)
    assert abs(sb["contacts"] - sa["contacts"]) < 0.35 * sa["contacts"]
