"""numpy model of ksg_update_esdf's incremental rule (csrc/ksg_esdf.cuh), built on the batch twin tests/esdf_ref.py.

update() takes the state the previous update stored (site bytes and outputs per block), the map as it is now (an export dict) and the
blocks touched since then, and returns the new state and the counts of ksg_esdf_stats:
  C = the touched blocks + the blocks new to the map;  R = C + its allocated face neighbours (their site bytes are recomputed);
  S = the blocks of R whose site bytes changed;  D = C + the allocated blocks within Chebyshev distance Rb = ceil(W / vps) of S;
  the outputs of D are recomputed from the stored site bytes of the whole map, every other output is kept.
Two mutants of the rule are parameters, so the tests can show their scenes tell them apart: `dilation` (a radius other than Rb) and
`face_neighbours=False` (R = C).  Test infrastructure."""
import math

import numpy as np

import esdf_ref as er

FACES = ((1, 0, 0), (-1, 0, 0), (0, 1, 0), (0, -1, 0), (0, 0, 1), (0, 0, -1))


def block_radius(voxel_size, vps, max_distance):
    return int(math.ceil(er.window(voxel_size, max_distance) / vps))


def _cells(bi, vps, lo):
    lin = np.arange(vps ** 3)
    l = np.stack([lin % vps, (lin // vps) % vps, lin // (vps * vps)], 1)
    return np.asarray(bi, np.int64)[:, None, :] * vps + l[None] - lo


def sites_by_block(exp, vps, min_weight=1e-4):
    """{block (x, y, z): site bytes [V] bool} of the whole map, by the kernel's site rule"""
    lo, obs, dist, _ = er.dense(exp, vps, min_weight)
    s = er.sites(obs, dist)
    g = _cells(exp["block_index"], vps, lo)
    return {tuple(int(c) for c in b): s[g[i, :, 0], g[i, :, 1], g[i, :, 2]] for i, b in enumerate(exp["block_index"])}


def work_sets(alloc, has_site, out, Rb):
    """(x_blocks, y_blocks): sizes of the x and y work sets EsdfWork::build makes for the z work set `out`"""
    near_x = {(b[0] + k, b[1], b[2]) for b in alloc if has_site[b] for k in range(-Rb, Rb + 1)}
    ys = set()
    for a in out:
        for k in range(-Rb, Rb + 1):
            b = (a[0], a[1], a[2] + k)
            if b not in ys and any((b[0], b[1] + j, b[2]) in near_x for j in range(-Rb, Rb + 1)):
                ys.add(b)
    xs = {(y[0], y[1] + j, y[2]) for y in ys for j in range(-Rb, Rb + 1)} & near_x
    return len(xs), len(ys)


def update(state, exp, changed, voxel_size, vps, max_distance, min_weight=1e-4, dilation=None, face_neighbours=True):
    """state: None (no update yet) or what the last call returned; changed: blocks touched since then.  -> (state, stats); the state's
    "out" maps each block to (distance [V] f32, flags [V] u8)"""
    keys = [tuple(int(c) for c in b) for b in np.asarray(exp["block_index"]).reshape(-1, 3)]
    alloc = set(keys)
    V = vps ** 3
    full = state is None or state["params"] != (float(min_weight), float(max_distance))
    old_sites = {} if full else state["sites"]
    old_out = {} if full else state["out"]
    C = set(alloc) if full else ({tuple(int(c) for c in b) for b in changed} & alloc) | (alloc - set(old_sites))
    R = set(C)
    if face_neighbours:
        for b in C:
            R |= {(b[0] + f[0], b[1] + f[1], b[2] + f[2]) for f in FACES} & alloc
    now = sites_by_block(exp, vps, min_weight)
    sites = {b: old_sites[b] for b in alloc if b in old_sites}
    S = set()
    for b in R:
        before = sites.get(b, np.zeros(V, bool))
        if (before != now[b]).any():
            S.add(b)
        sites[b] = now[b]
    W = er.window(voxel_size, max_distance)
    Rb = int(math.ceil(W / vps))
    r = Rb if dilation is None else dilation
    D = set(C)
    if S and keys:
        A = np.array(keys, np.int64)
        Sa = np.array(sorted(S), np.int64)
        near = (np.abs(A[:, None, :] - Sa[None, :, :]).max(axis=2) <= r).any(axis=1)
        D |= {keys[i] for i in np.flatnonzero(near)}
    out = {b: old_out[b] for b in alloc if b in old_out}
    if D:
        lo, obs, dist, _ = er.dense(exp, vps, min_weight)
        site = np.zeros_like(obs)
        g = _cells(keys, vps, lo)
        for i, b in enumerate(keys):
            site[g[i, :, 0], g[i, :, 1], g[i, :, 2]] = sites[b]
        dgrid, fgrid = er.finish(obs, dist, site, er.squared(site, W), voxel_size, max_distance)
        for i, b in enumerate(keys):
            if b in D:
                out[b] = (dgrid[g[i, :, 0], g[i, :, 1], g[i, :, 2]], fgrid[g[i, :, 0], g[i, :, 1], g[i, :, 2]])
    has_site = {b: bool(sites[b].any()) for b in alloc}
    nx, ny = work_sets(alloc, has_site, D, Rb) if D else (0, 0)
    stats = {"blocks": len(alloc), "full": int(full), "changed_blocks": len(C), "site_blocks": len(R), "site_changed": len(S),
             "x_blocks": nx, "y_blocks": ny, "z_blocks": len(D)}
    return {"params": (float(min_weight), float(max_distance)), "sites": sites, "out": out, "D": D}, stats


def as_export(state, blocks=None):
    """the state's outputs as ksg_export_esdf returns them: every block, or `blocks`, in (z, y, x) order"""
    keys = sorted(state["out"] if blocks is None else blocks, key=lambda b: (b[2], b[1], b[0]))
    V = len(next(iter(state["out"].values()))[0]) if state["out"] else 1
    return {"block_index": np.array(keys, np.int32).reshape(-1, 3),
            "distance": np.array([state["out"][b][0] for b in keys], np.float32).reshape(-1, V),
            "flags": np.array([state["out"][b][1] for b in keys], np.uint8).reshape(-1, V)}


def esdf_query(layer, voxel_size, vps, xyz):
    """twin of ksg_query_esdf on an exported layer (export_esdf()): the TSDF point-query twin (tests/query_ref.py) run on the ESDF
    distance, with "observed" = KSG_ESDF_OBSERVED, plus the containing voxel's ESDF flags and distance"""
    import query_ref as qr
    fake = {"block_index": layer["block_index"], "tsdf_distance": layer["distance"],
            "tsdf_weight": ((layer["flags"] & er.OBSERVED) != 0).astype(np.float32)}
    q = qr.query(fake, voxel_size, vps, xyz, min_weight=0.0)
    out = {"flags": q["flags"], "distance": q["distance"], "gradient": q["gradient"]}
    m = qr._Map(fake, voxel_size, vps, 0.0)
    p = np.ascontiguousarray(xyz, np.float32).reshape(-1, 3)
    valid = m.in_range(p)
    g = m.grid_index(np.where(valid[:, None], p, np.float32(0)))
    valid &= qr._key_in_range(m.block_of_voxel(g))
    row, lin = m.voxel(g)
    have = valid & (row >= 0)
    r = np.where(have, row, 0)
    fl = np.asarray(layer["flags"]).reshape(len(layer["block_index"]), -1) if len(layer["block_index"]) else np.zeros((1, vps ** 3), np.uint8)
    dd = np.asarray(layer["distance"]).reshape(len(layer["block_index"]), -1) if len(layer["block_index"]) else qr.nan((1, vps ** 3))
    out["voxel_flags"] = np.where(have, fl[r, lin], 0).astype(np.uint8)
    out["voxel_distance"] = np.where(have, dd[r, lin], qr.nan(len(p))).astype(np.float32)
    return out
