"""Plain-Python restatement of the batch scheduler (nudge.cpp:4206-4340, `k_schedule` in nb_solver.cuh) and of its segmented
replay (`k_sched_spec` / `k_sched_join` / `k_schedule` / `k_sched_merge`), used to show that the two give the same schedule.

Contacts are in tag order; contact i belongs to bucket i % 16 and has bucket-local index m = i // 16.  Per bucket the scheduler
keeps a list of partially filled 8-lane slots: a contact goes to the first slot holding neither of its bodies (a new slot at the
end of the list if there is none), a slot that receives its 8th contact is complete and the last slot of the list takes its
place.  A slot's id is the bucket-local index of the contact that opened it.  Completed slots are emitted in the order of the
contact that completed them (over all buckets); the slots still open at the end follow, bucket by bucket, in list order."""
import numpy as np

NONE = None


class Slot:
    __slots__ = ("uid", "bodies", "fill")

    def __init__(self, uid, bodies=(), fill=0):
        self.uid, self.bodies, self.fill = uid, set(bodies), fill

    def copy(self):
        return Slot(self.uid, self.bodies, self.fill)


class Overflow(Exception):
    """The list grew past the positions a run may hold."""


def replay(pairs, lo, hi, state, slot_of, done, empty_after=None, stop=None, cap=None):
    """First-fit over the bucket contacts lo..hi-1 starting from `state` (a list of Slot, modified in place).  Writes
    slot_of[m] = (uid, lane) and done[uid] (None while open, the completing m once complete).  `empty_after` (a set) collects
    the m after which the list is empty.  With `stop` (a predicate on m), the replay stops after the first m after which the list
    is empty and stop(m) holds and returns that m; it returns None when it ran to hi.  `cap`: largest list length (Overflow beyond)."""
    for m in range(lo, hi):
        a, b = pairs[m]
        for j, s in enumerate(state):
            if a not in s.bodies and b not in s.bodies:
                break
        else:
            if cap is not None and len(state) >= cap:
                raise Overflow()
            j = len(state)
            state.append(Slot(m))
            done[m] = NONE
        s = state[j]
        slot_of[m] = (s.uid, s.fill)
        s.fill += 1
        s.bodies.update((a, b))
        if s.fill == 8:
            done[s.uid] = m
            state[j] = state[-1]
            state.pop()
        if not state:
            if empty_after is not None:
                empty_after.add(m)
            if stop is not None and stop(m):
                return m
    return None


def sequential(pairs):
    """One bucket, one run from the empty list: (slot_of, done, leftover list)."""
    n = len(pairs)
    slot_of, done, state = [None] * n, {}, []
    replay(pairs, 0, n, state, slot_of, done)
    return slot_of, done, state


def segment_bounds(n, segs, seg_len):
    return [(min(k * seg_len, n), min((k + 1) * seg_len, n)) for k in range(segs)]


def segmented(pairs, segs, seg_len, cap=None, stats=None, join_cap=64, phases=8):
    """The segmented replay of one bucket.
    Speculative runs: for every segment k and r = 0..phases-1 (r = 0 only for the first segment), run r replays the segment from
    the empty list starting r contacts after the segment start.
    Joins: for every segment k >= 1 and every run r_in of segment k-1, segment k is replayed from the end state of run r_in until
    the first contact t after which its list is empty and speculative run r = (t + 1 - start) mod 8 either starts at t + 1 or has
    an empty list after t as well; from t + 1 on, run r is the true run if r_in was.  A join may replay at most `join_cap` contacts.
    (Every slot holds 8 contacts, so a list that is empty after t and was empty before contact c has placed a multiple of 8
    contacts since c: runs can only meet where they started a multiple of 8 apart, hence the 8 phases.)
    The chain of picks from run 0 of segment 0 gives the true run of every segment.  Falls back to `sequential` when a join on
    the chain does not couple or a list outgrows `cap`.  Returns (slot_of, done, leftover list, fell_back).  `stats` (a dict)
    receives the lengths of the joins on the chain."""
    n = len(pairs)
    bounds = segment_bounds(n, segs, seg_len)
    try:
        runs = {}
        for k, (lo, hi) in enumerate(bounds):
            for r in range(phases if k else 1):
                if lo + r > hi:
                    continue
                so, st, ea = {}, [], set()
                replay(pairs, lo + r, hi, st, so, {}, empty_after=ea, cap=cap)
                runs[k, r] = (so, st, ea)
        joins = {}
        for k in range(1, segs):
            lo, hi = bounds[k]
            for rin in range(phases if k > 1 else 1):
                if (k - 1, rin) not in runs:
                    continue
                st = [s.copy() for s in runs[k - 1, rin][1]]
                t, js = lo - 1, {}
                if st:
                    def stop(m, lo=lo, k=k):
                        q = m + 1 - lo
                        return q < min(phases, 8) or (q % 8 < phases and m in runs[k, q % 8][2])
                    t = replay(pairs, lo, min(hi, lo + join_cap), st, js, {}, stop=stop, cap=cap)
                joins[k, rin] = None if t is None else (t + 1 - lo, (t + 1 - lo) % 8, js)
        slot_of = [None] * n
        r = 0
        for m in range(*bounds[0]):
            slot_of[m] = runs[0, 0][0][m]
        for k in range(1, segs):
            lo, hi = bounds[k]
            j = joins.get((k, r))
            if j is None:
                raise Overflow()   # the join on the chain did not couple: the bucket falls back
            jn, r, js = j
            if stats is not None and jn:
                stats.setdefault("join_len", []).append(jn)
            for m in range(lo, lo + jn):
                slot_of[m] = js[m]
            for m in range(lo + jn, hi):
                slot_of[m] = runs[k, r][0][m]
        done = {}
        for m, (uid, lane) in enumerate(slot_of):
            if lane == 7:
                done[uid] = m
        left = runs[segs - 1, r][1] if segs else []
        for s in left:
            done[s.uid] = NONE
    except Overflow:
        s, d, left = sequential(pairs)
        return s, d, left, True
    return slot_of, done, left, False


def resolve(n, per_bucket):
    """Global schedule from per-bucket (slot_of, done, leftover list): batch and lane of every contact i."""
    complete = np.zeros(n, np.int64)
    for bkt, (slot_of, done, _) in enumerate(per_bucket):
        for m, (uid, lane) in enumerate(slot_of):
            if lane == 7:
                complete[bkt + 16 * m] = 1
    off = np.cumsum(complete) - complete
    nfull = int(complete.sum())
    left_base = np.concatenate([[0], np.cumsum([len(pb[2]) for pb in per_bucket])])
    batch = np.zeros(n, np.int64); lane_of = np.zeros(n, np.int64)
    for bkt, (slot_of, done, left) in enumerate(per_bucket):
        pos = {s.uid: p for p, s in enumerate(left)}
        for m, (uid, lane) in enumerate(slot_of):
            i = bkt + 16 * m
            t = done[uid]
            batch[i] = off[bkt + 16 * t] if t is not None else nfull + left_base[bkt] + pos[uid]
            lane_of[i] = lane
    return batch, lane_of


def buckets(cab):
    """cab: (n, 2) body pairs in tag order -> 16 lists of (ca, cb) tuples."""
    cab = np.asarray(cab).reshape(-1, 2)
    return [[(int(a), int(b)) for a, b in cab[k::16]] for k in range(16)]


def schedule_sequential(cab):
    bs = buckets(cab)
    return resolve(len(np.asarray(cab).reshape(-1, 2)), [sequential(p) for p in bs])


def schedule_segmented(cab, segs, seg_len, cap=None, stats=None, phases=8):
    """Returns (batch, lane, number of fallen-back buckets)."""
    bs = buckets(cab)
    res = [segmented(p, segs, seg_len, cap=cap, stats=stats, phases=phases) for p in bs]
    batch, lane = resolve(len(np.asarray(cab).reshape(-1, 2)), [r[:3] for r in res])
    return batch, lane, sum(r[3] for r in res)


def body_pairs(bodies_sorted):
    """(ca, cb) of every contact from its (body a, body b) in tag order, with the body-0 substitution of nudge.cpp:4238-4240."""
    ab = np.asarray(bodies_sorted, np.int64).reshape(-1, 2)
    ca = np.where(ab[:, 0] != 0, ab[:, 0], ab[:, 1]); cb = np.where(ab[:, 1] != 0, ab[:, 1], ab[:, 0])
    return np.stack([ca, cb], 1)
