"""The voxels a `fast` frame updates, defined without the CUDA path: the reference for the update log of the fast integrator.

Neither a map diff nor a fresh oracle can serve.  A diff misses the voxels whose update changed nothing (a voxel at max_weight and
+truncation seen again by a label-0 point).  And which voxels a `fast` frame updates depends on the integrator's two approximate sets,
which carry over from frame to frame (fast.h:114-130), so a fresh integrator casts different rays.  The trace therefore comes from the
LIVE oracle that integrates beside the device.  With its fast trace switched on (kso_trace_fast), the oracle records, for every ray it
casts, the point index and the number of voxels the ray updated before it ended or broke on collisions (ks_oracle.cpp:500-519).  That
ray's updated voxels are the first `updates` voxels of the same RayCaster walk, which kso_raycast replays.
tests/test_fast_update_trace_cpu.py checks this definition against an independent numpy replay and against the oracle's counters,
map and updated() blocks."""
import ctypes as C

import numpy as np

from kimera_semantics_b200 import synth
from kimera_semantics_b200.capi import _ptr
from parity_utils import frames

F = np.float32


def enable(ora):
    """Switch on the per-ray trace of a live OracleIntegrator (before its next frame)."""
    ora.lib.kso_get_fast_trace.argtypes = [C.c_void_p, C.c_int64, C.POINTER(C.c_int64), C.POINTER(C.c_int64)]
    ora.lib.kso_get_fast_trace.restype = C.c_int64
    ora.lib.kso_trace_fast.argtypes = [C.c_void_p, C.c_int]
    ora.lib.kso_trace_fast.restype = None
    ora.lib.kso_trace_fast(ora.handle, 1)


def rays(ora):
    """(point index [R], updates [R]) of every ray the oracle's last frame cast, in cast order."""
    n = int(ora.lib.kso_get_fast_trace(ora.handle, 0, None, None))
    idx, upd = np.zeros(n, np.int64), np.zeros(n, np.int64)
    if n:
        ora.lib.kso_get_fast_trace(ora.handle, n, _ptr(idx, C.c_int64), _ptr(upd, C.c_int64))
    return idx, upd


def depth_cloud(ora, depth, K):
    """kso_backproject's cloud of a depth image: the points (and point indices) the oracle's integrate_depth integrates."""
    depth = np.ascontiguousarray(depth, F)
    K = np.ascontiguousarray(K, F)
    h, w = depth.shape
    xyz, pix = np.zeros((h * w, 3), F), np.zeros(h * w, np.int32)
    n = int(ora.lib.kso_backproject(_ptr(depth, C.c_float), w, h, _ptr(K, C.c_float), _ptr(xyz, C.c_float), _ptr(pix, C.c_int32)))
    return xyz[:n], pix[:n]


def is_clearing(cfg, xyz, freespace):
    """isPointValid's clearing flag (A.6) of every point: a freespace frame, or a range beyond max_ray_length_m with allow_clear
    (which the voxblox constructor switches off when carving is off)."""
    x, y, z = (np.asarray(xyz, F)[:, k] for k in range(3))
    rng = np.sqrt(((x * x + y * y) + z * z).astype(F)).astype(F)
    allow_clear = bool(cfg.allow_clear) and bool(cfg.voxel_carving_enabled)
    return np.full(len(rng), bool(freespace)) | (allow_clear & (rng > F(cfg.max_ray_length_m)))


def records(ora, cfg, T, xyz, freespace=False):
    """Global voxel index [U, 3] of every voxel update of the oracle's last `fast` frame (integrate_points(T, xyz, freespace)), ray by ray
    in cast order (U = voxel_updates), and the clearing flag [R] and full walk length [R] of every cast ray (a ray that updated fewer
    voxels than its walk broke on collisions)."""
    lib = ora.lib
    idx, upd = rays(ora)
    xyz = np.ascontiguousarray(xyz, F)
    T = np.ascontiguousarray(T, F)
    origin = np.ascontiguousarray(T[4:], F)
    clear = is_clearing(cfg, xyz, freespace)[idx]
    vsi = F(1.0 / float(F(cfg.voxel_size)))          # voxblox: 1.0 / voxel_size in double, stored as float (A.1)
    trunc, max_len = F(cfg.default_truncation_distance), F(cfg.max_ray_length_m)
    carving = int(cfg.voxel_carving_enabled)
    out = np.zeros((int(upd.sum()), 3), np.int64)
    walks = np.zeros(len(idx), np.int64)
    pG = np.zeros(3, F)
    at = 0
    for r, (i, n, c) in enumerate(zip(idx.tolist(), upd.tolist(), clear.tolist())):
        lib.kso_transform(_ptr(T, C.c_float), _ptr(xyz[i], C.c_float), _ptr(pG, C.c_float))
        buf = out[at:at + n]
        walked = lib.kso_raycast(_ptr(origin, C.c_float), _ptr(pG, C.c_float), int(c), carving, max_len, vsi, trunc, 0,
                                 _ptr(buf, C.c_int64), n)
        assert walked >= n, (i, walked, n)
        walks[r] = walked
        at += n
    return out, clear, walks


def block_lin(vox, vps):
    """Global voxel indices [n, 3] -> (block index [n, 3], voxblox linear index x + vps*(y + vps*z) [n])."""
    vox = np.asarray(vox, np.int64).reshape(-1, 3)
    b = np.floor_divide(vox, vps)
    loc = vox - b * vps
    return b, loc[:, 0] + vps * (loc[:, 1] + vps * loc[:, 2])


def pairs(block_index, lin):
    """A set of (bx, by, bz, linear index) tuples."""
    bi = np.asarray(block_index, np.int64).reshape(-1, 3)
    return set(zip(bi[:, 0].tolist(), bi[:, 1].tolist(), bi[:, 2].tolist(), np.asarray(lin, np.int64).tolist()))


# ---- the frame sequences of the fast update-log tests ------------------------------------------------------------------------------

def sequence(W, H, C, seed=0, colours=False, n_depth=2, all_label0=False):
    """(kind, args) frames: n_depth depth frames, the points of the next frame with explicit labels (and random point colours with
    `colours`), then the points of one more frame integrated as freespace points.  At C = 256 label 1 becomes label 255 (the top bits of
    lin_label); `all_label0` replaces every label by 0 (the likelihood column of label 0 is zero: the row does not move)."""
    out = []
    fr = list(frames(W, H, C, n_depth + 2, seed=seed))
    for k, (cam, depth, label, T) in enumerate(fr):
        if C == 256:
            label = np.where(label == 1, 255, label).astype(np.uint8)
        if all_label0:
            label = np.zeros_like(label)
        if k < n_depth:
            out.append(("depth", (T, depth, label, cam.K)))
            continue
        xyz, pix = synth.backproject(depth, cam)
        lab = np.ascontiguousarray(label.reshape(-1)[pix], np.uint8)
        rgba = None
        if colours and k == n_depth:
            rgba = np.random.default_rng(seed + 7).integers(0, 256, (len(xyz), 4)).astype(np.uint8)
        out.append(("freespace" if k == n_depth + 1 else "points", (T, xyz, lab, rgba)))
    return out


def integrate(x, kind, args):
    """One frame of `sequence` into an Integrator or an OracleIntegrator."""
    if kind == "depth":
        return x.integrate_depth(*args)
    T, xyz, labels, rgba = args
    return x.integrate_points(T, xyz, rgba=rgba, labels=labels, freespace=(kind == "freespace"))


def frame_records(ora, cfg, kind, args):
    """records() of the frame `kind, args` the live oracle just integrated."""
    if kind == "depth":
        T, depth, _label, K = args
        return records(ora, cfg, T, depth_cloud(ora, depth, K)[0])
    T, xyz, _labels, _rgba = args
    return records(ora, cfg, T, xyz, freespace=(kind == "freespace"))
