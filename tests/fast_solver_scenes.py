"""Hand-built `fast` scenes that drive the observed-set solver (k_fast_solve3, ksg_fast3.cuh) down its rare paths, each with a
certificate computed on the CPU that proves the scene reaches its path.

A builder returns (cfg, frames, cert).  A frame is (T_G_C, points_C, labels, freespace) for integrate_points; everything is
seeded.  The certificate comes from the numpy restatement of the `fast` control flow (test_oracle_crosscheck.py), the ray lists of
test_fixpoint_prototype.py and the solver model of tools/observed_set_fixpoint.py, never from the device:

1. aliased start cells: two start cells whose index hashes are equal mod 2^20 share one start-set slot; more than kSortPerWarp
   = 1024 visitors make phase 0b sort the slot's visitors in global memory instead of shared memory;
2. overflowing buckets: rays that do not stop converge on the camera, so the voxels next to it collect far more than kBkt3 = 32
   entries and the overflow chain is used; the second case also reaches voxels 75 cells apart that alias into those slots;
3. window edges: long rays (1 cm voxels, 3-4 m) that break at steps 63, 64, 65, 127 and 128, on both sides of the 64-step
   evaluation blocks;
4. deep fixpoint: a planar fan whose Jacobi iteration needs many sweeps, so the device's worklist runs;
5. persistence: scenes 2-4 run three frames from overlapping poses, so that the persistent table decides collisions.
"""
import os
import sys
from collections import Counter

import numpy as np

from kimera_semantics_b200.capi import KSG_INTEGRATOR_FAST, KSG_ORDER_MIXED
from parity_utils import make_config
from test_fixpoint_prototype import cast_rays_of_frame
from test_oracle_crosscheck import ApproxSet, f32, grid_index, index_hash, norm, transform

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))
import observed_set_fixpoint as fx  # noqa: E402

BUCKET = 32                 # kBkt3: bucket entries per observed-set slot
SORT_PER_WARP = 1024        # kSortPerWarp: visitors of a shared start-set slot sorted in shared memory
WINDOW = 64                 # kWin: steps per evaluation block past step 64
WINDOW_EDGE_STEPS = (63, 64, 65, 127, 128)
ALIAS = (75, -61, 0)        # 75 + 17191 * (-61) = -2^20: cells this far apart share a slot of either approximate set
C = 5                       # labels; label C - 1 is dynamic (make_config)


def pose(tx=0.0, ty=0.0, tz=0.0):
    return np.array([1, 0, 0, 0, tx, ty, tz], np.float32)


def off_axis(xyz):
    """Moves exactly-zero coordinates to 1 mm.  With the camera at a pose without rotation, a point with a zero coordinate casts a
    ray with an exactly zero component, whose RayCaster divides 0 by 0 (SURVEY.md A.7): the walk then repeats one voxel, and the
    result is unspecified in the reference as well (INTEGRATION.md), so no scene may contain one."""
    xyz = np.array(xyz, np.float64)
    xyz[np.abs(xyz) < 1e-4] = 1e-3
    return xyz


def overflow_cap(cfg):
    """ovf_cap of ksg_create: the overflow pool shared by every slot of a frame."""
    return min(max(1 << 20, 4 * int(cfg.max_points)), 1 << 28)


def certify(cfg, frames):
    """The CPU model of every frame in order; the start set and the observed-set table persist across frames as in the
    integrator.  Per frame: ray lengths, the sequential U, the Jacobi sweeps from the device's start min(L, max collisions),
    the bucket entries per slot, the collisions the persistent table decides and the points whose ray has an exactly zero
    component (see off_axis)."""
    maxc = int(cfg.max_consecutive_ray_collisions)
    start_set = ApproxSet()
    table = {0: (1 << 64) - 1}
    out = []
    for offset, (T, xyz, labels, _) in enumerate(frames, start=1):
        start_set.reset()
        rays = cast_rays_of_frame(cfg, T, xyz, labels, start_set, offset)
        origin = T[4:].astype(np.float32)
        zero = sum(bool((transform(T, p) - origin == 0).any()) for p in xyz)
        U, table_after = fx.sequential(rays, table, maxc)
        U_jacobi, sweeps = fx.solve(rays, table, maxc, [min(len(r), maxc) for r in rays])
        assert U_jacobi == U
        entries = fx.slot_entries(rays, U)
        counts = [len(v) for v in entries.values()]
        out.append({"rays": len(rays), "lengths": [len(r) for r in rays], "U": U, "sweeps": sweeps,
                    "candidates": sum(len(r) for r in rays), "max_entries": max(counts, default=0),
                    "slots_over_bucket": sum(c > BUCKET for c in counts),
                    "mixed_slots_over_bucket": sum(len(v) > BUCKET and len(set(v)) > 1 for v in entries.values()),
                    "table_collisions": fx.table_collisions(rays, table, U), "zero_ray_components": zero})
        table = table_after
    return out


def start_slot_visitors(cfg, T, xyz, labels):
    """(visitors, distinct start cells) of the busiest start-set slot that several cells share."""
    vsi = f32(1.0 / f32(cfg.voxel_size))
    start_inv = f32(f32(cfg.start_voxel_subsampling_factor) * vsi)
    visitors, cells = Counter(), {}
    for p, lab in zip(xyz, labels):
        rng = norm(p)
        if rng < f32(cfg.min_ray_length_m) or rng > f32(cfg.max_ray_length_m) or cfg.dynamic_label[int(lab)]:
            continue
        g = grid_index(transform(T, p), start_inv)
        slot = index_hash(g) & fx.MASK
        visitors[slot] += 1
        cells.setdefault(slot, set()).add(g)
    shared = [s for s in visitors if len(cells[s]) > 1]
    if not shared:
        return 0, 0
    s = max(shared, key=lambda k: visitors[k])
    return visitors[s], len(cells[s])


# ---------------------------------------------------------------------------------------------------------------------------
# 1. aliased start cells
# ---------------------------------------------------------------------------------------------------------------------------
START_VISITORS = (1023, 1024, 1025, 3000)


def scene_aliased_start(order=KSG_ORDER_MIXED, visitors=START_VISITORS, seed=1, certificate=True):
    """One frame per visitor count.  Every point lies in one of two start cells ALIAS apart (2 cm voxels, 1 cm start cells,
    75 cm x 61 cm apart, 2 m in front of the camera); a handful of the second cell's points sit at evenly spread sequence positions, so visitors of the two
    cells alternate and a ray is cast at every change of cell."""
    vs = 0.02
    cfg = make_config(KSG_INTEGRATOR_FAST, vs, C, max_points=4096, integration_order_mode=order)
    cell = 1.0 / float(f32(f32(cfg.start_voxel_subsampling_factor) * f32(1.0 / f32(vs))))    # start cells are 1 cm
    a = np.array([-37, 30, 200])
    b = a + np.array(ALIAS)
    rng = np.random.default_rng(seed)
    frames = []
    for n in visitors:
        k = 8
        in_b = np.zeros(n, bool)
        in_b[np.linspace(n // (2 * k), n - 1, k).astype(int)] = True
        corner = np.where(in_b[:, None], b, a).astype(np.float64) * float(cell)
        xyz = (corner + rng.uniform(0.15, 0.85, (n, 3)) * float(cell)).astype(np.float32)
        labels = rng.integers(0, C - 1, n).astype(np.uint8)
        frames.append((pose(), xyz, labels, False))
    if not certificate:
        return cfg, frames, None
    cert = certify(cfg, frames)
    for c, (T, xyz, labels, _) in zip(cert, frames):
        c["start_slot_visitors"], c["start_slot_cells"] = start_slot_visitors(cfg, T, xyz, labels)
    return cfg, frames, cert


# ---------------------------------------------------------------------------------------------------------------------------
# 2. overflowing buckets (three frames from overlapping poses)
# ---------------------------------------------------------------------------------------------------------------------------
def sphere_points(n, radius, seed):
    """n points on a Fibonacci sphere around the camera, radii jittered within +-2 %."""
    rng = np.random.default_rng(seed)
    i = np.arange(n) + 0.5
    z = 1 - 2 * i / n
    phi = np.pi * (1 + 5 ** 0.5) * i
    r = np.sqrt(1 - z * z)
    d = np.stack([r * np.cos(phi), r * np.sin(phi), z], 1)
    return (d * radius * rng.uniform(0.98, 1.02, (n, 1))).astype(np.float32)


def overlapping_poses(n, step):
    return [pose(step * k, -0.5 * step * k, 0.25 * step * k) for k in range(n)]


def scene_overflow(case="fan", n_frames=3, seed=2, certificate=True):
    """Rays from every direction converge on the camera and never stop (max_consecutive_ray_collisions = 1000), so the voxels
    next to the camera collect up to one entry per ray.  "fan": 2000 rays of 5 cm voxels ending 2-3 m away.  "alias": 3000
    rays that end 4.9 m away, past the cells ALIAS away from the voxels next to the camera, which share their slots."""
    vs = 0.05
    cfg = make_config(KSG_INTEGRATOR_FAST, vs, C, max_points=4096, max_consecutive_ray_collisions=1000)
    n, radius = (2000, 2.5) if case == "fan" else (3000, 4.9)
    rng = np.random.default_rng(seed)
    xyz = sphere_points(n, radius, seed)
    labels = rng.integers(0, C - 1, n).astype(np.uint8)
    frames = [(T, xyz, labels, False) for T in overlapping_poses(n_frames, 0.3 * vs)]
    return cfg, frames, certify(cfg, frames) if certificate else None


# ---------------------------------------------------------------------------------------------------------------------------
# 3. window edges
# ---------------------------------------------------------------------------------------------------------------------------
def _break_step(cfg, a, b):
    """U of ray b after ray a (a fresh frame): where b breaks on a's trace."""
    ss = ApproxSet()
    ss.reset()
    rays = cast_rays_of_frame(cfg, pose(), np.stack([a, b]).astype(np.float32), np.zeros(2, np.uint8), ss, 1)
    if len(rays) != 2:
        return None
    return fx.sequential(rays, {0: (1 << 64) - 1}, int(cfg.max_consecutive_ray_collisions))[0][1]


def _direction(az, el):
    return np.array([np.sin(az) * np.cos(el), np.sin(el), np.cos(az) * np.cos(el)])


def scene_window_edges(max_collisions, n_frames=3, origin=(0.0, 0.0, 0.0), certificate=True):
    """1 cm voxels.  For every step s of WINDOW_EDGE_STEPS a long ray B (3.5 m, ~500 steps) and, ranked before it, a ray A whose
    point lies on B's line closer to the camera: B runs onto A's trace and breaks there.  A's distance is searched in 1 mm
    steps until B breaks exactly at s.  The pairs are 0.12 rad apart, so they do not meet before they near the camera.  A fan
    of 200 rays below them (see scene_deep_fixpoint), ranked after them, makes the solver run past its third sweep.
    `origin` moves the camera (and the scene with it), e.g. to the edge of the voxel-index range."""
    vs = 0.01
    cfg = make_config(KSG_INTEGRATOR_FAST, vs, C, max_points=4096, max_consecutive_ray_collisions=max_collisions)
    As, Bs = [], []
    for g, s in enumerate(WINDOW_EDGE_STEPS):
        u = _direction(-0.3 + 0.12 * g, 0.05 + 0.03 * g)
        b = u * 3.5
        lo, hi = 0.05, 1.6                       # the break step grows with A's distance from B's point: bisect, then scan
        for _ in range(16):
            mid = 0.5 * (lo + hi)
            if (_break_step(cfg, u * (3.5 - mid), b) or 0) < s:
                lo = mid
            else:
                hi = mid
        found = None
        for da in np.arange(lo - 0.01, lo + 0.02, 0.0005):
            if _break_step(cfg, u * (3.5 - da), b) == s:
                found = u * (3.5 - da)
                break
        assert found is not None, f"no point on the ray breaks it at step {s}"
        As.append(found)
        Bs.append(b)
    fan = fan_points(200, 3.0, 0.00334, -0.2)      # ranked after the pairs: long rays whose solution takes many sweeps
    xyz = np.concatenate([np.stack(As + Bs), fan]).astype(np.float32)
    labels = (np.arange(len(xyz)) % (C - 1)).astype(np.uint8)
    frames = [(pose(*(T[4:] + np.array(origin, np.float32))), xyz, labels, False) for T in overlapping_poses(n_frames, 0.3 * vs)]
    if not certificate:
        return cfg, frames, None
    cert = certify(cfg, frames)
    for c in cert:
        c["edge_hist"] = {s: c["U"].count(s) for s in WINDOW_EDGE_STEPS}
    return cfg, frames, cert


# ---------------------------------------------------------------------------------------------------------------------------
# 4. deep fixpoint
# ---------------------------------------------------------------------------------------------------------------------------
DEEP = dict(vs=0.02, max_collisions=0, n=200, distance=3.003, dtheta=0.00334, elevation=0.103)


def fan_points(n, distance, dtheta, elevation):
    """A fan of n points in rank order, azimuths dtheta apart and centred on the optical axis, at height sin(elevation) * distance."""
    th = dtheta * (np.arange(n) - 0.5 * n)
    return off_axis(np.stack([np.sin(th), np.full(n, np.sin(elevation)), np.cos(th)], 1) * distance)


def scene_deep_fixpoint(n_frames=3, certificate=True, **kw):
    """Ray r of the fan first meets rays r-1, r-2, ... at distances that shrink with the angle between them, so whether it
    reaches ray r-2 depends on how far ray r-1 ran: a chain of dependencies through the fan.  The parameters (DEEP) are the
    deepest Jacobi iteration a search over fans found."""
    p = dict(DEEP, **kw)
    cfg = make_config(KSG_INTEGRATOR_FAST, p["vs"], C, max_points=4096, max_consecutive_ray_collisions=p["max_collisions"])
    xyz = fan_points(p["n"], p["distance"], p["dtheta"], p["elevation"]).astype(np.float32)
    labels = (np.arange(len(xyz)) % (C - 1)).astype(np.uint8)
    frames = [(T, xyz, labels, False) for T in overlapping_poses(n_frames, 0.3 * p["vs"])]
    return cfg, frames, certify(cfg, frames) if certificate else None
