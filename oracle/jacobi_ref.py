"""CPU restatement of the THROUGHPUT-mode solver (nudge_b200/csrc/nb_jacobi.cuh) — TEST INFRASTRUCTURE ONLY.

Only tests/ may import this.  The throughput mode is not the reference's algorithm (the reference is sequential Gauss-Seidel,
/root/reference/nudge.cpp:4640-4855): it is a mass-splitting Jacobi iteration (Tonge, Benevolenski, Voroshilov, "Mass splitting for
jitter-free parallel rigid body simulation", SIGGRAPH 2012) whose PER-CONTACT arithmetic is the reference's — restated here in
float64 numpy from nudge.cpp:4646-4853 (one sweep of one contact) and nudge.cpp:4563-4632 (warm start), over the reference's own row
layout ContactConstraintV (nudge.cpp:907-957).  Parity status: the per-contact arithmetic is pinned indirectly — the same planes
and the same formulas are pinned bit-for-bit in parity mode (tests/test_gpu_parity.py); the Jacobi coupling itself has no
reference counterpart and is checked against this restatement within a tolerance plus physical invariants
(tests/test_gpu_throughput.py).

Row planes are passed as an array P[plane, contact] in the order of the enum in nb_solver.cuh (= member order of ContactConstraintV
plus the two inverse-mass planes)."""
import numpy as np

PLANES = ("PA_Z PA_X PA_Y PB_Z PB_X PB_Y N_X U_X V_X N_Y U_Y V_Y N_Z U_Z V_Z BIAS FRICTION NVTNI FC_X FC_Y FC_Z "
          "NA_X NA_Y NA_Z NB_X NB_Y NB_Z UA_X UA_Y UA_Z VA_X VA_Y VA_Z UB_X UB_Y UB_Z VB_X VB_Y VB_Z MASS_A MASS_B").split()
IX = {n: i for i, n in enumerate(PLANES)}


def _v(P, *names):
    return np.stack([P[IX[n]].astype(np.float64) for n in names], 1)


def split_terms(P, a, b, cnt):
    """Effective-mass planes of the mass split, recomputed from PARITY-mode rows (nudge.cpp:4350-4561 builds them unsplit).

    Body i counts cnt[i] contacts and is split into cnt[i] sub-bodies, so every per-body term of the effective masses is scaled by
    cnt[i] (body 0, the static world, has zero inverse mass and inertia).  Returns dict(NVTNI, BIAS, FC_X, FC_Y, FC_Z)."""
    sa = np.maximum(cnt[a], 1).astype(np.float64); sb = np.maximum(cnt[b], 1).astype(np.float64)
    pa, pb = _v(P, "PA_X", "PA_Y", "PA_Z"), _v(P, "PB_X", "PB_Y", "PB_Z")
    n, u, v = _v(P, "N_X", "N_Y", "N_Z"), _v(P, "U_X", "U_Y", "U_Z"), _v(P, "V_X", "V_Y", "V_Z")
    ma, mb = P[IX["MASS_A"]].astype(np.float64), P[IX["MASS_B"]].astype(np.float64)
    # the A-side planes are stored negated (nudge.cpp:4516-4534): I_a^-1 (pa x n) = -NA, etc.
    na, ua_t, va_t = -_v(P, "NA_X", "NA_Y", "NA_Z"), -_v(P, "UA_X", "UA_Y", "UA_Z"), -_v(P, "VA_X", "VA_Y", "VA_Z")
    nb, ub_t, vb_t = _v(P, "NB_X", "NB_Y", "NB_Z"), _v(P, "UB_X", "UB_Y", "UB_Z"), _v(P, "VB_X", "VB_Y", "VB_Z")
    dot = lambda x, y: (x * y).sum(1)
    ka = ma + dot(np.cross(na, pa), n); kb = mb + dot(np.cross(nb, pb), n)
    k = sa * ka + sb * kb
    nvtni = np.where(k != 0, -1.0 / np.where(k != 0, k, 1.0), 0.0)
    old = P[IX["NVTNI"]].astype(np.float64)
    bias = np.where(old != 0, P[IX["BIAS"]].astype(np.float64) / np.where(old != 0, old, 1.0) * nvtni, 0.0)
    ua, va_, ub, vb_ = np.cross(pa, u), np.cross(pa, v), np.cross(pb, u), np.cross(pb, v)
    fx = sa * (ma + dot(ua, ua_t)) + sb * (mb + dot(ub, ub_t))
    fy = sa * (ma + dot(va_, va_t)) + sb * (mb + dot(vb_, vb_t))
    fz = sa * 2.0 * dot(ua, va_t) + sb * 2.0 * dot(ub, vb_t)
    return dict(NVTNI=nvtni, BIAS=bias, FC_X=fx, FC_Y=fy, FC_Z=fz)


def _first_on_nan_min(x, y):
    """simd min(x, y) = (y < x) ? y : x: the first operand when y is NaN (nudge.cpp:286-289, 594-597)."""
    with np.errstate(invalid="ignore"):
        return np.where(y < x, y, x)


def jacobi_pass(P, states, a, b, lin, ang, warm=False, impulses=None, abs_sums=False):
    """One Jacobi pass over all contacts.  P[41, n] rows (split planes already in place), states[3, n] accumulated impulses,
    a/b body indices, lin/ang [B, 3] velocities at the START of the pass.  Returns (lin', ang', states').
    Per-contact arithmetic: nudge.cpp:4646-4853 (sweep) / 4563-4632 (warm start); coupling: every contact sees the start-of-pass
    velocities and the per-body changes are summed (Jacobi).

    abs_sums: also return (|dlin|, |dang|) [B, 3], the per-body sums of the absolute per-contact velocity changes.  They bound the
    rounding of a float32 sum whose order is free (the kernel's atomics): |error| <= (terms) * 2^-24 * sum of |terms|."""
    f = np.float64
    g = lambda n: P[IX[n]].astype(f)
    va, wa, vb, wb = lin[a].astype(f), ang[a].astype(f), lin[b].astype(f), ang[b].astype(f)
    n = _v(P, "N_X", "N_Y", "N_Z"); u = _v(P, "U_X", "U_Y", "U_Z"); v = _v(P, "V_X", "V_Y", "V_Z")
    NA, UA, VA = _v(P, "NA_X", "NA_Y", "NA_Z"), _v(P, "UA_X", "UA_Y", "UA_Z"), _v(P, "VA_X", "VA_Y", "VA_Z")
    NB, UB, VB = _v(P, "NB_X", "NB_Y", "NB_Z"), _v(P, "UB_X", "UB_Y", "UB_Z"), _v(P, "VB_X", "VB_Y", "VB_Z")
    ma, mb = g("MASS_A"), g("MASS_B")
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        if warm:  # nudge.cpp:4563-4632
            ci = impulses.astype(f)
            ni = np.maximum((n * ci).sum(1), 0.0)
            mf = ni * g("FRICTION")
            fx, fy = (u * ci).sum(1), (v * ci).sum(1)
            s = 1.0 / np.sqrt(fx * fx + fy * fy) * mf
            s = _first_on_nan_min(np.ones_like(s), s)
            fx, fy = fx * s, fy * s
            dn, dfx, dfy = ni, fx, fy
            new_states = np.stack([ni, fx, fy])
        else:     # nudge.cpp:4646-4853
            pa, pb = _v(P, "PA_X", "PA_Y", "PA_Z"), _v(P, "PB_X", "PB_Y", "PB_Z")
            rel = (vb + np.cross(wb, pb)) - (va + np.cross(wa, pa))   # the reference interleaves the cross products lane-wise (4682-4711)
            t_z, t_x, t_y = (n * rel).sum(1), (u * rel).sum(1), (v * rel).sum(1)
            old_n, old_fx, old_fy = states[0].astype(f), states[1].astype(f), states[2].astype(f)
            ni = np.maximum(g("NVTNI") * t_z + (g("BIAS") + old_n), 0.0)
            t_xx, t_yy, t_xy = t_x * t_x, t_y * t_y, t_x * t_y
            tl2 = t_xx + t_yy
            t_x, t_y = t_x * tl2, t_y * tl2
            mf = ni * g("FRICTION")
            dn = ni - old_n
            ff = 1.0 / (t_xx * g("FC_X") + t_yy * g("FC_Y") + t_xy * g("FC_Z"))
            ff = _first_on_nan_min(np.full_like(ff, 1e6), ff)
            fx, fy = old_fx - t_x * ff, old_fy - t_y * ff
            s = 1.0 / np.sqrt(fx * fx + fy * fy) * mf
            s = _first_on_nan_min(np.ones_like(s), s)
            fx, fy = fx * s, fy * s
            dfx, dfy = fx - old_fx, fy - old_fy
            new_states = np.stack([ni, fx, fy])
    J = n * dn[:, None] + u * dfx[:, None] + v * dfy[:, None]
    la, lb = -J * ma[:, None], J * mb[:, None]
    wa_, wb_ = NA * dn[:, None] + UA * dfx[:, None] + VA * dfy[:, None], NB * dn[:, None] + UB * dfx[:, None] + VB * dfy[:, None]
    dlin = np.zeros(lin.shape, f); dang = np.zeros(ang.shape, f)
    np.add.at(dlin, a, la); np.add.at(dlin, b, lb)
    np.add.at(dang, a, wa_); np.add.at(dang, b, wb_)
    dlin[0] = 0; dang[0] = 0   # body 0 is the static world
    out = (lin.astype(f) + dlin, ang.astype(f) + dang, new_states)
    if not abs_sums:
        return out
    alin = np.zeros(lin.shape, f); aang = np.zeros(ang.shape, f)
    np.add.at(alin, a, np.abs(la)); np.add.at(alin, b, np.abs(lb))
    np.add.at(aang, a, np.abs(wa_)); np.add.at(aang, b, np.abs(wb_))
    alin[0] = 0; aang[0] = 0
    return out + (alin, aang)
