"""numpy twin of ksg_compute_esdf (csrc/ksg_esdf.cuh): a padded dense grid of the exported map, the surface voxels (sites), three
windowed passes over x, y, z of integer squared offsets, and the outputs in export order.  float32 where the kernel rounds (sqrtf and
the product), integers everywhere else, so it equals the kernel bit for bit."""
import math

import numpy as np

F = np.float32
OBSERVED, SURFACE, CAPPED = 1, 2, 4
NAN_BITS = 0x7FC00000
NONE = np.int64(1) << 40


def window(voxel_size, max_distance):
    """W = ceil(m / vs) + 1, in double from the float32 inputs (as the host entry computes it)"""
    return int(math.ceil(float(F(max_distance)) / float(F(voxel_size)))) + 1


def dense(exp, vps, min_weight=1e-4):
    """(lo, observed, distance, allocated): grids [x, y, z] over the blocks' bounding box with one voxel of padding; lo = the global
    voxel index of grid cell (0, 0, 0)"""
    bi = np.asarray(exp["block_index"], np.int64)
    lo = bi.min(0) * vps - 1
    shape = tuple((bi.max(0) + 1) * vps + 1 - lo)
    obs = np.zeros(shape, bool)
    dist = np.zeros(shape, F)
    alloc = np.zeros(shape, bool)
    lin = np.arange(vps ** 3)
    l = np.stack([lin % vps, (lin // vps) % vps, lin // (vps * vps)], 1)
    for i, b in enumerate(bi):
        g = b * vps + l - lo
        d = np.asarray(exp["tsdf_distance"][i], F)
        w = np.asarray(exp["tsdf_weight"][i], F)
        dist[g[:, 0], g[:, 1], g[:, 2]] = d
        obs[g[:, 0], g[:, 1], g[:, 2]] = w > F(min_weight)
        alloc[g[:, 0], g[:, 1], g[:, 2]] = True
    return lo, obs, dist, alloc


def _shifted(a, axis, t, fill):
    """b[p] = a[p + t e_axis], `fill` outside the grid"""
    b = np.full_like(a, fill)
    n = a.shape[axis]
    if abs(t) >= n:
        return b
    src = [slice(None)] * 3
    dst = [slice(None)] * 3
    src[axis] = slice(max(t, 0), n + min(t, 0))
    dst[axis] = slice(max(-t, 0), n + min(-t, 0))
    b[tuple(dst)] = a[tuple(src)]
    return b


def sites(obs, dist):
    pos = dist > 0
    mag = np.abs(dist)
    s = np.zeros_like(obs)
    for axis in range(3):
        for t in (-1, 1):
            on = _shifted(obs, axis, t, False)
            pn = _shifted(pos, axis, t, False)
            mn = _shifted(mag, axis, t, F(0))
            s |= obs & on & (pos != pn) & (mag <= mn)
    return s


def squared(site, W):
    """Q: the three windowed passes (int64; NONE = no site in the window)"""
    a = np.full(site.shape, NONE, np.int64)
    for t in range(-W, W + 1):
        a = np.where(_shifted(site, 0, t, False), np.minimum(a, t * t), a)
    for axis in (1, 2):
        b = np.full(site.shape, NONE, np.int64)
        for t in range(-W, W + 1):
            s = _shifted(a, axis, t, NONE)
            b = np.minimum(b, np.where(s < NONE, s + t * t, NONE))
        a = b
    return a


def finish(obs, dist, site, Q, voxel_size, max_distance):
    """distance and flags grids from the sites and Q"""
    vs, m = F(voxel_size), F(max_distance)
    has = Q < NONE
    mag = np.sqrt(np.where(has, Q, 0).astype(F)) * vs
    capped = ~(has & (mag < m))
    mag = np.where(capped, m, mag).astype(F)
    out = np.where(dist > 0, mag, -mag).astype(F)
    out = np.where(site, dist, out)
    out = np.where(obs, out, np.array(NAN_BITS, np.uint32).view(F))
    flags = np.where(obs, OBSERVED | np.where(site, SURFACE, np.where(capped, CAPPED, 0)), 0).astype(np.uint8)
    return out.astype(F), flags


def esdf(exp, voxel_size, vps, max_distance, min_weight=1e-4, W=None):
    """{"block_index", "distance" (nb, V), "flags" (nb, V)} as ksg_compute_esdf returns them; W overrides the window (tests only)"""
    bi = np.asarray(exp["block_index"], np.int32).reshape(-1, 3)
    V = vps ** 3
    if len(bi) == 0:
        return {"block_index": bi, "distance": np.zeros((0, V), F), "flags": np.zeros((0, V), np.uint8)}
    W = window(voxel_size, max_distance) if W is None else W
    lo, obs, dist, _ = dense(exp, vps, min_weight)
    site = sites(obs, dist)
    out, flags = finish(obs, dist, site, squared(site, W), voxel_size, max_distance)
    lin = np.arange(V)
    l = np.stack([lin % vps, (lin // vps) % vps, lin // (vps * vps)], 1)
    g = bi.astype(np.int64)[:, None, :] * vps + l[None] - lo
    return {"block_index": bi, "distance": out[g[..., 0], g[..., 1], g[..., 2]],
            "flags": flags[g[..., 0], g[..., 1], g[..., 2]]}
