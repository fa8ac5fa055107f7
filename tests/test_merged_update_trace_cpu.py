"""The definition of "the voxels a merged frame updated" that the merged update-log tests compare against (merged_update_trace.py),
checked on the CPU against two independent descriptions of the same frames:

- a numpy restatement of bundling and the RayCaster (apply_edge_scenes.py), with anti-grazing (merged.cpp:306-313) restated here: the
  set of voxels its records visit must be the traced set, and its record count the oracle's voxel_updates;
- the oracle's own run of the frame on a live map: the traced voxels' blocks are its updated() blocks, the traced voxels hold every voxel
  whose state changed, and there are no more of them than updates."""
import numpy as np
import pytest

import apply_edge_scenes as S
import merged_update_trace as tr
from kimera_semantics_b200 import synth
from kimera_semantics_b200.capi import KSG_INTEGRATOR_MERGED
from oracle.oracle_py import OracleIntegrator
from parity_utils import make_config
from test_oracle_crosscheck import mixed_order

F = np.float32


def bundle_keys(cfg, T, xyz, freespace):
    """The grid voxel of every bundle of S.bundles_of_frame, in the same order."""
    t = T[4:].astype(F)
    xyz = np.asarray(xyz, F)
    rng = S.norm_rows(xyz)
    valid = ~(rng < F(cfg.min_ray_length_m))
    clearing = np.full(len(xyz), bool(freespace))
    far = rng > F(cfg.max_ray_length_m)
    if cfg.allow_clear or freespace:
        clearing |= far
    else:
        valid &= ~far
    vox = S.grid_rows((xyz + t).astype(F), F(1.0 / F(cfg.voxel_size)))
    seen, order = set(), []
    for i in mixed_order(len(xyz)):
        key = (bool(clearing[i]), tuple(vox[i]))
        if valid[i] and key not in seen:
            seen.add(key)
            order.append(key)
    order = [k for k in order if not k[0]] + [k for k in order if k[0]]
    return np.array([k[1] for k in order], np.int64).reshape(-1, 3)


def restated_records(cfg, T, xyz, freespace):
    """Voxels of the frame's update records [R, 3]: the numpy RayCaster, minus the steps anti-grazing drops."""
    origin = T[4:].astype(F)
    pG, _, bc = S.bundles_of_frame(cfg, T, xyz, freespace)
    ids, vox = S.raycast_many(cfg, origin, pG, bc)
    if cfg.enable_anti_grazing:
        keys = bundle_keys(cfg, T, xyz, freespace)
        nonclear = {tuple(k) for k in keys[~bc]}                 # voxel_keys = the non-clearing map (merged.cpp:306-313)
        own = (vox == keys[ids]).all(axis=1)
        end = np.array([tuple(v) in nonclear for v in vox.tolist()], bool)
        vox = vox[~((bc[ids] | ~own) & end)]
    return vox


def edge_frames():
    """(name, cfg, frames) of the rotation-free scenes, as merged scenes, with and without anti-grazing."""
    out = []
    for name, build in (("route_edge_n255", lambda: S.scene_route_edge(255, 21, certificate=False)),
                        ("moving_distance", lambda: S.scene_moving_distance("semantic", n=1500, certificate=False))):
        cfg, frames, _ = build()
        for ag in (0, 1):
            c = make_config(KSG_INTEGRATOR_MERGED, cfg.voxel_size, cfg.num_labels, max_points=cfg.max_points,
                            merged_bundle_order=cfg.merged_bundle_order, default_truncation_distance=cfg.default_truncation_distance,
                            max_weight=cfg.max_weight, use_const_weight=cfg.use_const_weight, enable_anti_grazing=ag)
            out.append((f"{name}_ag{ag}", c, frames))
    return out


@pytest.mark.parametrize("name,cfg,frames", edge_frames(), ids=lambda x: x if isinstance(x, str) else "")
def test_traced_voxels_equal_the_restated_raycaster_and_sum_to_voxel_updates(name, cfg, frames):
    ora = OracleIntegrator(cfg)
    freespace_seen = False
    for T, xyz, labels, freespace, rgba in frames:
        so = ora.integrate_points(T, xyz, rgba=rgba, labels=labels, freespace=freespace)
        vox = restated_records(cfg, T, xyz, freespace)
        assert len(vox) == so.voxel_updates, name
        got = tr.pairs(*tr.updated_voxels_points(cfg, T, xyz, freespace=freespace))
        assert got == tr.voxel_pairs(np.unique(vox, axis=0), cfg.voxels_per_side), name
        assert {p[:3] for p in got} == {tuple(b) for b in ora.last_updated_blocks().tolist()}, name
        freespace_seen |= bool(freespace)
    ora.close()
    assert name.startswith("route_edge") or freespace_seen


@pytest.mark.parametrize("anti_grazing", [0, 1])
def test_traced_voxels_cover_every_changed_voxel_and_the_updated_blocks_of_depth_frames(anti_grazing):
    """Rotating depth frames at 5 cm: the traced voxels' blocks are the oracle's updated() blocks, every voxel whose state changed on the
    live map is traced, and the traced voxels are at most the updates (a voxel takes one update per record)."""
    W, H, C = 96, 72, 21
    cfg = make_config(KSG_INTEGRATOR_MERGED, 0.05, C, max_points=W * H, enable_anti_grazing=anti_grazing)
    cam = synth.make_camera(W, H)
    ora = OracleIntegrator(cfg)
    before = None
    for f in range(3):
        depth, label, T = synth.frame(cam, f, C)
        so = ora.integrate_depth(T, depth, label, cam.K)
        exp = ora.export()
        bi, lin = tr.updated_voxels_depth(cfg, T, depth, cam.K)
        got = tr.pairs(bi, lin)
        assert 0 < len(got) <= so.voxel_updates
        assert {p[:3] for p in got} == {tuple(b) for b in ora.last_updated_blocks().tolist()}
        changed = set()
        for b, key in enumerate(map(tuple, exp["block_index"].tolist())):
            old = before.get(key) if before else None
            rows = np.concatenate([exp["sem_priors"][b].view(np.uint32), exp["tsdf_distance"][b].view(np.uint32)[:, None],
                                   exp["tsdf_weight"][b].view(np.uint32)[:, None]], axis=1)
            moved = np.ones(len(rows), bool) if old is None else (rows != old).any(axis=1)
            if old is None:    # a new block: only the voxels that left the constructor's state are known to be updated
                moved = (rows[:, :C] != tr.P_INIT.view(np.uint32)).any(axis=1) | (rows[:, C:] != 0).any(axis=1)
            changed |= {key + (int(v),) for v in np.flatnonzero(moved)}
        assert changed <= got
        before = {tuple(k): np.concatenate([exp["sem_priors"][b].view(np.uint32), exp["tsdf_distance"][b].view(np.uint32)[:, None],
                                            exp["tsdf_weight"][b].view(np.uint32)[:, None]], axis=1)
                  for b, k in enumerate(exp["block_index"].tolist())}
    ora.close()
