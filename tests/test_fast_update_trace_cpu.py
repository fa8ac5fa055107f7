"""The definition of "the voxels a fast frame updated" that the fast update-log tests compare against (fast_update_trace.py), checked on
the CPU for every frame of the sequences test_gpu_fast_update_log.py runs:

- the traced rays are the oracle's rays_cast and their update counts sum to its voxel_updates;
- the traced set equals the set of FastReplay (test_oracle_crosscheck.py), an independent numpy restatement of fast.cpp's control flow
  that shares no code with the oracle;
- the traced set holds every voxel whose state changed on the live map, and its blocks are the oracle's updated() blocks.

Certificates make the comparisons mean something: one scene updates voxels without changing them (so the set is more than a map diff),
and the sequences reach collision breaks, start-set rejections and clearing rays."""
import numpy as np
import pytest

import fast_update_trace as ft
from oracle.oracle_py import OracleIntegrator
from test_gpu_fast_update_log import CASES, H, W, fast_config
from test_oracle_crosscheck import FastReplay

P_INIT = np.float32(-0.60205999132)


def voxel_state(exp):
    """{(bx, by, bz): [V, k] uint32 rows} of distance, weight, label and log-probabilities."""
    rows = np.concatenate([exp["tsdf_distance"].view(np.uint32)[..., None], exp["tsdf_weight"].view(np.uint32)[..., None],
                           exp["sem_label"].astype(np.uint32)[..., None], exp["sem_priors"].view(np.uint32)], axis=2)
    return {tuple(b): rows[i] for i, b in enumerate(exp["block_index"].tolist())}


def changed(before, after, C):
    """(bx, by, bz, lin) of every voxel whose state differs; a new block starts from the constructor's state."""
    out = set()
    for key, rows in after.items():
        old = before.get(key)
        if old is None:
            old = np.zeros_like(rows)
            old[:, 3:] = P_INIT.view(np.uint32)
        out |= {key + (int(v),) for v in np.flatnonzero((rows != old).any(axis=1))}
    return out


def frames_of(name):
    ckw, skw, event = CASES[name]
    cfg = fast_config(**ckw)
    seq = ft.sequence(W, H, cfg.num_labels, **skw)
    if name == "saturated":
        seq = [seq[0], seq[0]]
    return cfg, seq, event


def replay_frame(rep, ora, kind, args):
    if kind == "depth":
        T, depth, label, K = args
        xyz, pix = ft.depth_cloud(ora, depth, K)
        return rep.integrate(T, xyz, label.reshape(-1)[pix])
    T, xyz, labels, _ = args
    return rep.integrate(T, xyz, labels, freespace=(kind == "freespace"))


@pytest.mark.parametrize("name", list(CASES))
def test_traced_voxels_equal_the_replay_counters_and_cover_every_change(name):
    cfg, seq, event = frames_of(name)
    vps, C = cfg.voxels_per_side, cfg.num_labels
    ora, rep = OracleIntegrator(cfg), FastReplay(cfg)
    ft.enable(ora)
    cert = dict(unchanged=0, breaks=0, start_rejections=0, clearing=0, label255=0)
    state = {}
    for f, (kind, args) in enumerate(seq):
        if f == 2 and event == "clear_map":
            ora.clear_map()
            state = {}
        elif f == 2 and event == "reset":
            ora.close()
            ora, rep = OracleIntegrator(cfg), FastReplay(cfg)
            ft.enable(ora)
            state = {}
        so = ft.integrate(ora, kind, args)
        vox, clear, walks = ft.frame_records(ora, cfg, kind, args)
        idx, upd = ft.rays(ora)
        where = f"{name} frame {f} ({kind})"
        assert len(idx) == so.rays_cast and int(upd.sum()) == so.voxel_updates == len(vox), where
        got = ft.pairs(*ft.block_lin(vox, vps))
        assert 0 < len(got) <= so.voxel_updates, where
        valid, rays, updates = replay_frame(rep, ora, kind, args)
        assert (valid, rays, updates) == (so.points_valid, so.rays_cast, so.voxel_updates), where
        assert got == ft.pairs(*ft.block_lin(np.array(sorted(rep.frame_touched), np.int64), vps)), where
        assert {p[:3] for p in got} == {tuple(b) for b in ora.last_updated_blocks().tolist()}, where
        exp = ora.export()
        now = voxel_state(exp)
        moved = changed(state, now, C)
        assert moved <= got, (where, len(moved - got))
        state = now
        cert["unchanged"] = max(cert["unchanged"], len(got - moved))
        cert["breaks"] += int((upd < walks).sum())
        cert["start_rejections"] += so.points_valid - so.rays_cast
        cert["clearing"] += int(clear.sum())
        cert["label255"] += int((exp["sem_label"] == 255).sum())
    assert cert["start_rejections"] > 0 and cert["clearing"] > 0, cert
    if name == "saturated":            # label 0 through voxels at max_weight and +truncation: updated, unchanged
        assert cert["unchanged"] > 1000, cert
    if name in ("base", "collisions0"):
        assert cert["breaks"] > 1000, cert
    if C == 256:
        assert cert["label255"] > 0, cert
    ora.close()


def test_the_dense_tile_scene_is_traced_exactly():
    from test_gpu_fast_voxel_items import scene
    cfg, fr = scene()
    ora, rep = OracleIntegrator(cfg), FastReplay(cfg)
    ft.enable(ora)
    for T, xyz, labels in fr:
        so = ft.integrate(ora, "points", (T, xyz, labels, None))
        vox = ft.frame_records(ora, cfg, "points", (T, xyz, labels, None))[0]
        assert rep.integrate(T, xyz, labels) == (so.points_valid, so.rays_cast, so.voxel_updates) and len(vox) == so.voxel_updates
        assert ft.pairs(*ft.block_lin(vox, 16)) == ft.pairs(*ft.block_lin(np.array(sorted(rep.frame_touched), np.int64), 16))
    ora.close()
