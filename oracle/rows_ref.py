"""CPU restatement of the user constraint rows (nudge_b200/csrc/nb_rows_api.cuh) — TEST INFRASTRUCTURE ONLY (tests/ imports it).

The reference has no such feature: it only marks where an application would apply its own constraint impulses
(/root/reference/example/main.cpp:316).  This is the sequential loop such an application would write at that line — plain sequential
impulses over generic velocity rows — in float64; the world-space inverse inertia follows nudge.cpp:4182-4199 (rotation matrix
nudge.cpp:1142-1163).  Parity unpinned against the reference (nothing to pin to); the GPU path is compared with this loop."""
import numpy as np


def world_inverse_inertia(rotation, inertia_inverse):
    """R diag(I^-1) R^T per body; rotation = (x, y, z, w) quaternions."""
    q = rotation.astype(np.float64)
    x, y, z, w = q[:, 0], q[:, 1], q[:, 2], q[:, 3]
    R = np.empty((len(q), 3, 3))
    R[:, 0, 0] = 1 - 2 * (y * y + z * z); R[:, 0, 1] = 2 * (x * y - z * w); R[:, 0, 2] = 2 * (x * z + y * w)
    R[:, 1, 0] = 2 * (x * y + z * w); R[:, 1, 1] = 1 - 2 * (x * x + z * z); R[:, 1, 2] = 2 * (y * z - x * w)
    R[:, 2, 0] = 2 * (x * z - y * w); R[:, 2, 1] = 2 * (y * z + x * w); R[:, 2, 2] = 1 - 2 * (x * x + y * y)
    return np.einsum("nij,nj,nkj->nik", R, inertia_inverse.astype(np.float64), R)


def apply_rows(rows, lin, ang, mass_inverse, inv_inertia, warm=False):
    """One pass over the rows in order (in place on lin, ang [B, 3] float64 and rows['impulse']).

    Rows with a == b != 0 are outside the model: their effective mass would need the cross terms 2 m lin_a.lin_b + 2 ang_a.I^-1 ang_b,
    which neither this loop nor the kernel computes; nb_upload_constraint_rows refuses them (put the whole Jacobian on a, b = 0)."""
    for r in rows:
        a, b = int(r["a"]), int(r["b"])
        la, aa, lb, ab = (r[k].astype(np.float64) for k in ("lin_a", "ang_a", "lin_b", "ang_b"))
        ma = mass_inverse[a] if a else 0.0; mb = mass_inverse[b] if b else 0.0
        Ia = inv_inertia[a] if a else np.zeros((3, 3)); Ib = inv_inertia[b] if b else np.zeros((3, 3))
        ia, ib = Ia @ aa, Ib @ ab
        if warm:
            delta = float(r["impulse"])
        else:
            k = ma * la @ la + aa @ ia + mb * lb @ lb + ab @ ib + float(r["softness"])
            jv = la @ lin[a] + aa @ ang[a] + lb @ lin[b] + ab @ ang[b]
            eff = 1.0 / k if k > 0 else 0.0
            nxt = float(r["impulse"]) - eff * (jv + float(r["bias"]) + float(r["softness"]) * float(r["impulse"]))
            nxt = min(max(nxt, float(r["lo"])), float(r["hi"]))
            delta = nxt - float(r["impulse"])
            r["impulse"] = nxt
        if a:
            lin[a] += ma * la * delta; ang[a] += ia * delta
        if b:
            lin[b] += mb * lb * delta; ang[b] += ib * delta
