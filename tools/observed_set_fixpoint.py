"""Reference model of how the CUDA path solves `fast`'s order-dependent observed-voxel set in parallel (DESIGN.md section 4),
small enough to read in one sitting and checked against the sequential definition in tests/test_fixpoint_prototype.py.

Sequential definition (fast.cpp:110-122 + ApproxHashSet::replaceHash, A.4): rays are processed in rank order; ray r walks its
voxels s = 0, 1, ...; at each step  collided = (table[slot] == value);  table[slot] = value;  the ray stops at the first step where
more than `max_collisions` collisions are consecutive, and every step before that updates its voxel.  U[r] = number of updated
voxels.  The table persists across frames.

Parallel formulation: a candidate (r, s) is PERFORMED iff s < U[r] or s is the breaking step itself (the breaking step still
executed replaceHash).  The slot always ends up holding the value of its latest visitor, so (r, s) collides iff the latest
performed candidate before it, in (rank, step) order, on the same slot carries the same value (none: the persistent table
decides).  U[r] depends only on rays of lower rank and on r's own earlier steps: a triangular system with a UNIQUE solution,
which plain Jacobi sweeps - re-evaluate every ray against the previous sweep's U - reach from ANY start in at most R + 1 sweeps
(in practice ~6-10 for a 640x480 frame, because a ray's outcome only depends on the few rays that share slots with it).
"""
from typing import Dict, List, Sequence, Tuple

MASK = (1 << 20) - 1


def sequential(rays: Sequence[Sequence[int]], table: Dict[int, int], max_collisions: int) -> Tuple[List[int], Dict[int, int]]:
    """rays[r] = values (hash + offset) of ray r's voxels in walking order. Returns (U, table after the frame)."""
    table = dict(table)
    U = []
    for vals in rays:
        run, n = 0, 0
        for v in vals:
            k = v & MASK
            if table.get(k) == v:
                run += 1
            else:
                run = 0
            table[k] = v
            if run > max_collisions:
                break
            n += 1
        U.append(n)
    return U, table


def visits(vals: Sequence[int], u: int) -> int:
    """Number of steps of a ray that execute replaceHash when it updates u voxels: the breaking step, if any, still does."""
    return min(len(vals), u + 1)


def jacobi_sweep(rays, table, max_collisions, U_prev, break_performed=True):
    """One parallel sweep: every ray is evaluated independently against the PREVIOUS estimate of all lower-ranked rays.
    break_performed=False leaves the breaking step out of the performed set, as the device does: it collided, so at the fixpoint
    its replaceHash rewrote the value the slot already held."""
    # per slot: performed candidates of the previous estimate as (rank, step, value), in (rank, step) order
    by_slot: Dict[int, List[Tuple[int, int, int]]] = {}
    for r, vals in enumerate(rays):
        for s in range(visits(vals, U_prev[r]) if break_performed else U_prev[r]):
            by_slot.setdefault(vals[s] & MASK, []).append((r, s, vals[s]))
    U_new = []
    for r, vals in enumerate(rays):
        run, n = 0, 0
        own: Dict[int, int] = {}                       # slot -> value of this ray's own latest earlier step (always performed)
        for s, v in enumerate(vals):
            k = v & MASK
            if k in own:
                prev = own[k]
            else:
                prev = table.get(k)
                for (r2, s2, v2) in by_slot.get(k, ()):   # latest performed visit by a lower-ranked ray
                    if r2 >= r:
                        break
                    prev = v2
            run = run + 1 if prev == v else 0
            own[k] = v
            if run > max_collisions:
                break
            n += 1
        U_new.append(n)
    return U_new


def solve(rays, table, max_collisions, U_start, max_sweeps=None):
    """Jacobi iteration to the fixpoint; returns (U, sweeps)."""
    U = list(U_start)
    limit = max_sweeps or len(rays) + 2
    for sweep in range(1, limit + 1):
        nxt = jacobi_sweep(rays, table, max_collisions, U)
        if nxt == U:
            return U, sweep
        U = nxt
    raise RuntimeError("no fixpoint within R + 2 sweeps: the system would not be triangular")


def examined(vals: Sequence[int], u: int) -> range:
    """Steps a ray that updates u voxels has looked at: the updated ones and the breaking step."""
    return range(min(len(vals), u + 1))


def slot_entries(rays, U) -> Dict[int, List[int]]:
    """Per slot, the values of the entries the device's solution leaves in its bucket (and overflow chain): every performed
    step and every breaking step, in (rank, step) order."""
    out: Dict[int, List[int]] = {}
    for vals, u in zip(rays, U):
        for s in examined(vals, u):
            out.setdefault(vals[s] & MASK, []).append(vals[s])
    return out


def table_collisions(rays, table, U) -> int:
    """Collisions of the solution that the persistent table decides: steps whose slot no earlier examined step of the frame
    visited, and whose value the table holds."""
    seen = set()
    n = 0
    for vals, u in zip(rays, U):
        for s in examined(vals, u):
            k = vals[s] & MASK
            if k not in seen and table.get(k) == vals[s]:
                n += 1
            seen.add(k)
    return n


def stamped_solve(rays, table, max_collisions, U_start, worklist: bool):
    """The device's iteration (ksg_fast3.cuh) on the Jacobi sweeps above.  A ray is re-evaluated only when it is DIRTY: never
    evaluated, or one of its examined slots was toggled (a step below U entered or left the performed set, or a breaking step
    entered the slot's bucket) in a later sweep
    than the ray's last evaluation, or in that sweep by another ray.  worklist=False tests every ray in every sweep; worklist=True
    tests only the scan list: every ray in sweep 1, then the rays evaluated in the previous sweep and every other ray with an entry in
    a slot the previous sweep toggled.  A slot's entries are the steps ever performed and the breaking steps, so every examined
    step can be found from its slot.
    Returns (U, sweeps, log) with one record per sweep: rays scanned, rays evaluated, dirty rays missing from the scan list, rays left
    clean whose evaluation would have changed them.  Exactness means the last two are always empty."""
    R = len(rays)
    U = list(U_start)
    last = [0] * R                                   # sweep of the last evaluation, 0 = never
    togglers: Dict[int, Dict[int, set]] = {}         # slot -> sweep -> rays that toggled it in that sweep
    entries: Dict[int, set] = {}                     # slot -> rays with an entry in it
    for r, vals in enumerate(rays):
        for s in range(min(len(vals), U[r])):
            entries.setdefault(vals[s] & MASK, set()).add(r)

    def dirty(r):
        if last[r] == 0:
            return True
        for s in examined(rays[r], U[r]):
            by_sweep = togglers.get(rays[r][s] & MASK, {})
            if any(k > last[r] for k in by_sweep) or by_sweep.get(last[r], set()) - {r}:
                return True
        return False

    scan = list(range(R))
    log = []
    for sweep in range(1, R + 3):
        dirty_now = {r for r in range(R) if dirty(r)}
        evaluated = [r for r in scan if r in dirty_now]
        nxt = jacobi_sweep(rays, table, max_collisions, U, break_performed=False)
        missing = sorted(dirty_now - set(scan))
        stale = [r for r in range(R) if r not in dirty_now and nxt[r] != U[r]]
        toggled: Dict[int, set] = {}
        changed_any = False
        for r in evaluated:
            vals, old, new = rays[r], U[r], nxt[r]
            changed_any |= new != old
            slots = {vals[s] & MASK for s in range(min(old, new), max(old, new))}
            if new < len(vals) and r not in entries.get(vals[new] & MASK, set()):
                slots.add(vals[new] & MASK)            # the breaking step enters the slot's bucket (a perf-0 entry)
            for k in slots:
                toggled.setdefault(k, set()).add(r)
                togglers.setdefault(k, {}).setdefault(sweep, set()).add(r)
            for s in examined(vals, new):
                entries.setdefault(vals[s] & MASK, set()).add(r)
            U[r] = new
            last[r] = sweep
        log.append((len(scan), len(evaluated), missing, stale))
        if not changed_any:
            return U, sweep, log
        if worklist:
            listed = set(evaluated)
            for k, by in toggled.items():
                listed |= {r2 for r2 in entries.get(k, ()) if by - {r2}}
            scan = sorted(listed)
    raise RuntimeError("no fixpoint within R + 2 sweeps")
