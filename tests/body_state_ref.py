"""Restatement of nb_get_body_states / nb_set_body_states (include/nudge_b200.h, DESIGN.md section 8.19) on host arrays, in numpy.

get_states(scene, bodies) is the gather; set_states(scene, rows, fields, cache_tags, kinematic) the host edit a set must equal, on a
scenes.Scene whose transforms, momentum and idle counters hold the current state: the fields in list order, idle counter 0 for every listed
dynamic body, and with BODY_POSE removal's wake (tests/spawn_ref.py, wake_set) with "removed" read as "moved".  valid(rows, fields, B) is
the check both call modes apply: the host path refuses a list with an invalid entry, the device path skips it."""
import numpy as np
from nudge_b200 import abi
from tests.spawn_ref import wake_set

REMOVED = np.uint32(0xffffffff)


def get_states(scene, bodies=None):
    """The BODY_STATE rows of `bodies` (None: 0 .. B-1); an index at or beyond B gives body = REMOVED and zeros."""
    B = scene.n_bodies
    idx = np.arange(B, dtype=np.uint32) if bodies is None else np.asarray(bodies, np.uint32).reshape(-1)
    out = np.zeros(len(idx), abi.BODY_STATE)
    ok = idx < B
    b = idx[ok].astype(np.int64)
    out["body"] = np.where(ok, idx, REMOVED)
    out["position"][ok] = scene.transforms["position"][b]; out["rotation"][ok] = scene.transforms["rotation"][b]
    out["velocity"][ok] = scene.momentum["velocity"][b]; out["angular_velocity"][ok] = scene.momentum["angular_velocity"][b]
    out["idle_counter"][ok] = scene.idle[b]
    return out


def valid(rows, fields, B):
    """Per entry: not body 0, below B, every selected field finite."""
    rows = np.asarray(rows, abi.BODY_STATE).reshape(-1)
    ok = (rows["body"] != 0) & (rows["body"] < B)
    sel = []
    if fields & abi.BODY_POSE:
        sel += ["position", "rotation"]
    if fields & abi.BODY_VELOCITY:
        sel += ["velocity", "angular_velocity"]
    for f in sel:
        ok &= np.isfinite(rows[f]).all(1)
    return ok


def set_states(scene, rows, fields, cache_tags=None, kinematic=()):
    """Returns (the edited scene, a copy, and the mask of bodies the call gave idle counter 0).  rows must all be valid; cache_tags = the
    contact cache's keys (u64 tags); kinematic = the context's kinematic bodies."""
    rows = np.asarray(rows, abi.BODY_STATE).reshape(-1)
    assert valid(rows, fields, scene.n_bodies).all()
    out = scene.copy()
    t, m = out.transforms, out.momentum
    for r in rows:
        b = int(r["body"])
        if fields & abi.BODY_POSE:
            t["position"][b] = r["position"]; t["rotation"][b] = r["rotation"]
        if fields & abi.BODY_VELOCITY:
            m["velocity"][b] = r["velocity"]; m["angular_velocity"][b] = r["angular_velocity"]
    listed = np.zeros(scene.n_bodies, bool)
    listed[rows["body"].astype(np.int64)] = True
    woken = listed.copy()
    if fields & abi.BODY_POSE:
        woken |= wake_set(scene, ~listed, cache_tags)
    woken[0] = False
    woken[np.asarray(kinematic, np.int64)] = False
    out.idle[woken] = 0
    return out, woken
