"""Hand-built scenes that put real voxels into the states where the voxel-update kernels switch paths (ksg_voxel.cuh, tsdf_batch in
ksg_kernels.cuh, k_tile_apply_fast), each with a certificate computed on the CPU that proves the scene reaches what it is named for.

A builder returns (cfg, frames, certificate).  A frame is (T_G_C, points_C, labels, freespace, rgba or None) for integrate_points;
everything is seeded.  The camera never rotates and no ray has an exactly zero component (fast_solver_scenes.off_axis).

The construction: with voxel carving every bundle's ray starts in the camera's voxel, so that voxel receives exactly one update record
per bundle.  N points in N distinct voxels on a shell around the camera therefore give it a segment of exactly N records, and the
voxels around it large fractions of N: a segment length, and with it the kernel route (k_voxel_heads: short / long / hot), can be set to
the record.  The same pose integrated again starts the same segments from the weights the last frame left.

The certificate of a `merged` scene comes from a vectorised numpy float32 restatement of bundling, the RayCaster and tsdf_measure (the
serial restatement in test_oracle_crosscheck.py is the check of the RayCaster) and the branch model of apply_branch_model.py: per frame
the record count of every voxel, and for the tracked voxels (>= TRACK_LEN records) the batches on each weight / distance path, per
route.  It is valid for KSG_BUNDLE_ORDER_CANONICAL, which the scenes set; route counts do not depend on the bundle order."""
from collections import Counter

import numpy as np

import apply_branch_model as M
from fast_solver_scenes import off_axis, pose
from kimera_semantics_b200 import synth
from kimera_semantics_b200.capi import KSG_BUNDLE_ORDER_CANONICAL, KSG_COLOR_MODE_COLOR, KSG_INTEGRATOR_FAST, KSG_INTEGRATOR_MERGED
from parity_utils import make_config
from test_oracle_crosscheck import mixed_order

F = np.float32
EPS = F(1e-6)
HOT_LEN = 4096              # kHotLen
TRACK_LEN = 32              # voxels with at least one full batch are followed through the branch model


def long_len(num_labels, env_long_len=None):
    """ksg_create: segments of at least this many records are `long` (thread-per-voxel short kernel at C <= 32, else warp-per-voxel)."""
    if num_labels <= 32:
        return 256 if env_long_len is None else max(96, min(1 << 20, env_long_len))
    return 96


def routes(lengths, llen):
    """Voxels per route from the histogram {segment length: voxels}."""
    out = Counter()
    for n, k in lengths.items():
        out["hot" if n >= llen and n >= HOT_LEN else "long" if n >= llen else "short"] += k
    return {r: out[r] for r in ("hot", "long", "short")}


# ---------------------------------------------------------------------------------------------------------------------------
# numpy float32 restatement of a merged frame, vectorised over rays
# ---------------------------------------------------------------------------------------------------------------------------
def norm_rows(v):
    return np.sqrt(((v[:, 0] * v[:, 0] + v[:, 1] * v[:, 1]).astype(F) + v[:, 2] * v[:, 2]).astype(F)).astype(F)


def grid_rows(p, inv):
    return np.floor(((p * inv).astype(F) + EPS).astype(F)).astype(np.int64)


def bundles_of_frame(cfg, T, xyz, freespace):
    """bundleRays + the merge loop (SURVEY.md A.5): (point_G [B,3], weight [B], clearing [B]) in canonical bundle order."""
    assert tuple(T[:4]) == (1, 0, 0, 0), "the scenes do not rotate the camera"
    t = T[4:].astype(F)
    vsi = F(1.0 / F(cfg.voxel_size))
    xyz = np.asarray(xyz, F)
    rng = norm_rows(xyz)
    valid = ~(rng < F(cfg.min_ray_length_m))
    clearing = np.full(len(xyz), bool(freespace))
    far = rng > F(cfg.max_ray_length_m)
    if cfg.allow_clear or freespace:
        clearing |= far
    else:
        valid &= ~far
    if cfg.use_const_weight:
        w = np.ones(len(xyz), F)
    else:
        z = np.abs(xyz[:, 2])
        with np.errstate(divide="ignore"):
            w = np.where(z > EPS, (F(1.0) / (z * z).astype(F)).astype(F), F(0.0)).astype(F)
    vox = grid_rows((xyz + t).astype(F), vsi)
    groups, order = {}, []
    for seq, i in enumerate(mixed_order(len(xyz))):
        if not valid[i]:
            continue
        key = (bool(clearing[i]), tuple(vox[i]))
        if key not in groups:
            groups[key] = []
            order.append(key)
        groups[key].append(i)
    order = [k for k in order if not k[0]] + [k for k in order if k[0]]        # the non-clearing map is integrated first
    pG, bw, bc = np.zeros((len(order), 3), F), np.zeros(len(order), F), np.zeros(len(order), bool)
    for b, key in enumerate(order):
        mp, mw = np.zeros(3, F), F(0.0)
        for i in groups[key]:
            if w[i] < EPS:
                continue
            tot = F(mw + w[i])
            mp = (((mp * mw).astype(F) + (xyz[i] * w[i]).astype(F)).astype(F) / tot).astype(F)
            mw = tot
            if key[0]:
                break                                                           # a clearing bundle takes its first point only
        pG[b], bw[b], bc[b] = (mp + t).astype(F), mw, key[0]
    return pG, bw, bc


def raycast_many(cfg, origin, pG, clearing):
    """RayCaster (A.7) from the camera for every bundle at once.  Returns (bundle id [R], voxel [R,3]) in (step, bundle) order."""
    vsi, trunc, max_len = F(1.0 / F(cfg.voxel_size)), F(cfg.default_truncation_distance), F(cfg.max_ray_length_m)
    assert cfg.voxel_carving_enabled
    d = (pG - origin).astype(F)
    n = norm_rows(d)
    unit = (d / n[:, None]).astype(F)
    L = np.minimum(np.maximum((n - trunc).astype(F), F(0)), max_len).astype(F)
    end = np.where(clearing[:, None], (origin + (unit * L[:, None]).astype(F)).astype(F), (pG + (unit * trunc).astype(F)).astype(F))
    s, e = np.broadcast_to((origin * vsi).astype(F), end.shape), (end * vsi).astype(F)
    cur = np.floor((s + EPS).astype(F)).astype(np.int64)
    endi = np.floor((e + EPS).astype(F)).astype(np.int64)
    steps = np.abs(endi - cur).sum(axis=1)
    r = (e - s).astype(F)
    sign = (r > 0).astype(np.int64) - (r < 0).astype(np.int64)
    with np.errstate(divide="ignore", invalid="ignore"):
        tn = ((np.maximum(0, sign).astype(F) - (s - cur.astype(F)).astype(F)).astype(F) / r).astype(F)
        ts = (sign.astype(F) / r).astype(F)
    ids, vox = [], []
    rows = np.arange(len(pG))
    for step in range(int(steps.max()) + 1):
        act = steps >= step
        ids.append(rows[act])
        vox.append(cur[act].copy())
        k = np.zeros(len(pG), np.int64)
        k[tn[:, 1] < tn[:, 0]] = 1
        k[tn[:, 2] < tn[rows, k]] = 2
        cur[rows, k] += sign[rows, k]
        tn[rows, k] = (tn[rows, k] + ts[rows, k]).astype(F)
    return np.concatenate(ids), np.concatenate(vox)


def measure(cfg, origin, pG, w, centers):
    """tsdf_measure per record: (sdf, update weight)."""
    trunc, vs = F(cfg.default_truncation_distance), F(cfg.voxel_size)
    vo, po = (centers - origin).astype(F), (pG - origin).astype(F)
    dist_G = norm_rows(po)
    dot = ((vo[:, 0] * po[:, 0] + vo[:, 1] * po[:, 1]).astype(F) + vo[:, 2] * po[:, 2]).astype(F)
    sdf = (dist_G - (dot / dist_G).astype(F)).astype(F)
    uw = w.astype(F).copy()
    if cfg.use_weight_dropoff:
        drop = sdf < -vs
        uw[drop] = np.maximum(((w[drop] * (trunc + sdf[drop]).astype(F)).astype(F) / F(trunc - vs)).astype(F), F(0.0))
    if cfg.use_sparsity_compensation_factor:
        near = np.abs(sdf) < trunc
        uw[near] = (uw[near] * F(cfg.sparsity_compensation_factor)).astype(F)
    return sdf, uw


def certify(cfg, frames, wide_hot=True):
    """Per frame: bundles, records, {segment length: voxels}, the camera voxel's segment, the zero-weight tail records, and for the
    tracked voxels the batches per (route, weight path, distance path) with the state carried from frame to frame."""
    llen = long_len(cfg.num_labels)
    blend = cfg.color_mode == KSG_COLOR_MODE_COLOR
    state, seen, out = {}, set(), []
    for T, xyz, _labels, freespace, _rgba in frames:
        origin = T[4:].astype(F)
        pG, bw, bc = bundles_of_frame(cfg, T, xyz, freespace)
        ids, vox = raycast_many(cfg, origin, pG, bc)
        centers = ((vox.astype(F) + F(0.5)) * F(cfg.voxel_size)).astype(F)
        sdf, uw = measure(cfg, origin, pG[ids], bw[ids], centers)
        key = (vox[:, 0] << 42) + (vox[:, 1] << 21) + vox[:, 2] + (1 << 62)    # one integer per voxel
        srt = np.lexsort((ids, key))                                            # per voxel, records in bundle order
        key_s = key[srt]
        heads = np.flatnonzero(np.r_[True, key_s[1:] != key_s[:-1]])
        lens = np.diff(np.r_[heads, len(key_s)])
        cam = tuple(grid_rows(origin[None, :], F(1.0 / F(cfg.voxel_size)))[0])
        cam_key = (cam[0] << 42) + (cam[1] << 21) + cam[2] + (1 << 62)
        first = np.zeros(len(key_s), bool)
        first[heads] = True
        fresh = np.array([k not in seen for k in key_s[heads]])
        zero_tail = int((first & np.repeat(fresh, lens) & (uw[srt] < EPS)).sum())
        seen.update(key_s[heads].tolist())
        paths = Counter()
        for h, n in zip(heads[lens >= TRACK_LEN], lens[lens >= TRACK_LEN]):
            sl = srt[h:h + n]
            route = "hot" if n >= HOT_LEN else "long" if n >= llen else "short"
            st = state.get(int(key_s[h]), (F(0), F(0), 0))
            d, wg, c, p, _ = M.batch_walk(cfg.default_truncation_distance, cfg.max_weight, route == "hot" and wide_hot, sdf[sl], uw[sl], None, blend, *st)
            state[int(key_s[h])] = (d, wg, c)
            for (wp, dp), cnt in p.items():
                paths[f"{route}/{wp}/{dp}"] += cnt
        out.append({"bundles": len(pG), "records": len(ids), "lengths": Counter(lens.tolist()), "routes": routes(Counter(lens.tolist()), llen),
                    "camera_voxel_records": int(lens[key_s[heads] == cam_key].sum()), "camera_voxel": cam,
                    "camera_voxel_state": state.get(int(cam_key)), "zero_weight_tail_records": zero_tail, "paths": dict(paths)})
    return out


# ---------------------------------------------------------------------------------------------------------------------------
# scenes
# ---------------------------------------------------------------------------------------------------------------------------
VS = 0.05
CAMERA = pose(0.5 * VS + 0.003, 0.5 * VS - 0.004, 0.5 * VS + 0.002)      # near the middle of its voxel


def shell_points(n, radius, seed, voxel_size=VS, T=CAMERA):
    """n points in n distinct voxels on a shell around the camera (Fibonacci sphere without the band |z| < 0.3 r, where the point
    weight 1 / z^2 would let a handful of points outweigh the rest; radii jittered within +-1 %)."""
    rng = np.random.default_rng(seed)
    m = 5 * n + 64
    i = np.arange(m) + 0.5
    z = 1 - 2 * i / m
    i, z = i[np.abs(z) >= 0.3], z[np.abs(z) >= 0.3]
    m = len(z)
    phi = np.pi * (1 + 5 ** 0.5) * i
    r = np.sqrt(1 - z * z)
    d = np.stack([r * np.cos(phi), r * np.sin(phi), z], 1) * radius * rng.uniform(0.99, 1.01, (m, 1))
    d = off_axis(d[rng.permutation(m)]).astype(F)
    vox = grid_rows((d + T[4:].astype(F)).astype(F), F(1.0 / F(voxel_size)))
    _, firsts = np.unique(vox, axis=0, return_index=True)
    keep = np.sort(firsts)[:n]
    assert len(keep) == n, "the shell has too few voxels"
    return d[keep]


def labels_for(n, C, seed):
    return np.random.default_rng(seed).integers(0, C, n).astype(np.uint8)


def merged_cfg(C, n_points, **kw):
    return make_config(KSG_INTEGRATOR_MERGED, VS, C, max_points=max(4096, n_points), merged_bundle_order=KSG_BUNDLE_ORDER_CANONICAL, **kw)


ROUTE_EDGES = {21: (255, 256, 257, 4095, 4096, 4097, 4128, 4160), 33: (95, 96, 97)}


def scene_route_edge(n, C, certificate=True):
    """One frame whose camera voxel holds exactly n records: the short / long / hot decision of k_voxel_heads at its thresholds, the
    batch count of the deep pipelines mod 3 and a last batch of 1, 31 and 32 records."""
    cfg = merged_cfg(C, n)
    frames = [(CAMERA, shell_points(n, 1.5, n), labels_for(n, C, n), False, None)]
    return cfg, frames, certify(cfg, frames) if certificate else None


WEIGHT_VARIANTS = {"default": {}, "const_weight": {"use_const_weight": 1}, "no_dropoff": {"use_weight_dropoff": 0},
                   "sparsity": {"use_sparsity_compensation_factor": 1, "sparsity_compensation_factor": 10.0},
                   "low_max_weight": {"use_const_weight": 1, "max_weight": 50.0}}


def scene_weight_states(variant="default", n=4200, C=21, certificate=True):
    """The same pose three times.  max_weight is 0.6 x the weight one frame adds to the camera voxel: frame 0 starts that voxel at
    weight 0 and crosses the clamp in the middle of its hot segment, frames 1 and 2 start it saturated at (+truncation, max_weight);
    the voxels around it saturate one after the other.  "low_max_weight" (50) saturates the short segments as well."""
    kw = dict(WEIGHT_VARIANTS[variant])
    low = kw.pop("max_weight", None)
    xyz, labels = shell_points(n, 1.5, 7), labels_for(n, C, 7)
    probe = merged_cfg(C, n, **kw)
    _, bw, _ = bundles_of_frame(probe, CAMERA, xyz, False)
    cfg = merged_cfg(C, n, max_weight=low or float(F(0.6 * float(bw.sum(dtype=np.float64)))), **kw)
    frames = [(CAMERA, xyz, labels, False, None)] * 3
    return cfg, frames, certify(cfg, frames) if certificate else None


MOVING_VARIANTS = {"semantic": (1, 2500.0, 3), "color": (0, 1e4, 2), "color_low_max_weight": (0, 40.0, 2)}


def scene_moving_distance(variant="semantic", n=4097, C=21, certificate=True):
    """Truncation distance 1.4 m around a shell of 1.25 m: the camera voxel and the voxels around it have |sdf| < truncation, so the
    distance moves on almost every record of their long segments (the replay path), at max_weight 2500 (the hot segment saturates in
    frame 0, the long ones in frame 2), 10^4 (bare chain to the last, partial batch) and 40 (short segments saturate too).  Then a
    shell at 3 m outside the truncation distance (pinned again once the mean is back at +truncation), and a freespace frame whose
    clearing rays pass the first surface."""
    color_mode, max_weight, n_near = MOVING_VARIANTS[variant]
    cfg = merged_cfg(C, n, default_truncation_distance=1.4, color_mode=color_mode, max_weight=max_weight, use_const_weight=1)
    near, lab = shell_points(n, 1.25, 9), labels_for(n, C, 9)
    frames = [(CAMERA, near, lab, False, None)] * n_near
    frames += [(CAMERA, (near * F(2.4)).astype(F), lab, False, None), (CAMERA, (near * F(3.6)).astype(F), lab, True, None)]
    return cfg, frames, certify(cfg, frames) if certificate else None


CLASS_COUNTS = (2, 31, 32, 33, 64, 65, 256)


def class_count_frames(C, seed=5):
    cam = synth.make_camera(96, 72)
    frames = []
    for f in range(2):
        depth, label, T = synth.frame(cam, f, C, seed=seed)
        xyz, pix = synth.backproject(depth, cam)
        frames.append((np.asarray(T, F), xyz, label.reshape(-1)[pix].astype(np.uint8), False, None))
    return frames


def scene_class_count(C, integrator=KSG_INTEGRATOR_MERGED, certificate=True):
    """The hot shell (4097 records on the camera voxel, labels over the whole range) and two frames of a small depth sequence at a
    class count where the kernels change: 2, the padded row table of the thread-per-voxel kernel with and without padding (31, 32),
    the switch to the warp-per-voxel kernels (33), two and three register chunks per lane (64, 65), the maximum (256)."""
    n = 4097
    if integrator == KSG_INTEGRATOR_MERGED:
        cfg = merged_cfg(C, 96 * 72)
    else:
        cfg = make_config(KSG_INTEGRATOR_FAST, VS, C, max_points=96 * 72)
    frames = [(CAMERA, shell_points(n, 1.5, 13), labels_for(n, C, C), False, None)]
    frames += class_count_frames(C)
    cert = None
    if certificate and integrator == KSG_INTEGRATOR_MERGED:
        cert = certify(cfg, frames[:1])            # the depth frames rotate the camera: their routes are counted on the device only
    return cfg, frames, cert


def scene_fast_saturate(certificate=True):
    """`fast`, ColorMode::kColor with a colour per point, max_weight 3: the same three poses again and again until the voxels
    saturate, through k_tile_apply_fast's tsdf_batch with real colours.  No certificate of paths: the CPU test asserts on the
    oracle's map that voxels reach max_weight and that colours were blended."""
    n, C = 3000, 21
    cfg = make_config(KSG_INTEGRATOR_FAST, VS, C, max_points=4096, color_mode=KSG_COLOR_MODE_COLOR, max_weight=3.0, use_const_weight=1,
                      max_consecutive_ray_collisions=1000)
    xyz = shell_points(n, 1.0, 17)
    rng = np.random.default_rng(17)
    labels = rng.integers(0, C - 1, n).astype(np.uint8)
    rgba = rng.integers(0, 256, (n, 4)).astype(np.uint8)
    poses = [pose(*(CAMERA[4:] + F(0.3 * VS * k) * F([1, -0.5, 0.25]))) for k in range(3)]
    frames = [(poses[k % 3], xyz, labels, False, rgba) for k in range(9)]
    return cfg, frames, None


def all_scenes(certificate=True):
    """(name, builder) of every scene, in a fixed order."""
    out = []
    for C, ns in ROUTE_EDGES.items():
        out += [(f"route_edge_n{n}_c{C}", lambda n=n, C=C, **k: scene_route_edge(n, C, **k)) for n in ns]
    out += [(f"weight_states_{v}", lambda v=v, **k: scene_weight_states(v, **k)) for v in WEIGHT_VARIANTS]
    out += [(f"moving_distance_{v}", lambda v=v, **k: scene_moving_distance(v, **k)) for v in MOVING_VARIANTS]
    out += [(f"class_count_merged_c{C}", lambda C=C, **k: scene_class_count(C, KSG_INTEGRATOR_MERGED, **k)) for C in CLASS_COUNTS]
    out += [(f"class_count_fast_c{C}", lambda C=C, **k: scene_class_count(C, KSG_INTEGRATOR_FAST, **k)) for C in CLASS_COUNTS]
    out += [("fast_saturate", scene_fast_saturate)]
    return out
