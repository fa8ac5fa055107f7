"""The update log of the `fast` integrator (written by k_fast_apply in ksg_fast.cuh, entry i = work item i): one entry per voxel the
frame updated, with the voxel's final state.  The eager host-layer sync of the C++ shim and the voxel-granular frame-batch merge
(ksg_merge_voxels_device) write only what the log lists, so a missing entry leaves a host layer or a merged replica stale.

The voxels a frame updated come from the live oracle that integrates beside the device (fast_update_trace.py, checked on the CPU by
test_fast_update_trace_cpu.py).  The cases reach every instantiation of the apply kernel (NCH = ceil(C / 32) = 1, 2, 4, 8), every
voxels_per_side from 2 to 32, the three colour modes, both point orders, collision breaks, carried-over approximate sets, spatial shards
and a tile of more than 4096 records.  Every comparison of state is bit for bit, except the colour of ColorMode::kSemanticProbability
(rainbow(expf(...)): +-1 per channel, as in test_gpu_parity.py)."""
import ctypes as ct
import os
import subprocess

import numpy as np
import pytest

import delta_merge_ref as dm
import fast_update_trace as ft
from kimera_semantics_b200 import synth
from kimera_semantics_b200.capi import (Integrator, KSG_COLOR_MODE_COLOR, KSG_COLOR_MODE_SEMANTIC_PROBABILITY, KSG_INTEGRATOR_FAST,
                                        KSG_ORDER_SORTED, owner_mask)
from oracle.oracle_py import OracleIntegrator
from parity_utils import assert_parity, compare_maps, frames, make_config
from test_gpu_more import read_shim_output
from test_shim_cpu import demo, write_frames  # noqa: F401

pytestmark = pytest.mark.gpu
W, H = 160, 120
KSG_ERR_SCRATCH_FULL = 4
GROUP_ROUND = 512           # k_fast_group reserves log slots once per 512 sorted records of a tile
LOG = 1 << 21


def fast_config(vs=0.05, C=21, vps=16, **kw):
    cfg = make_config(KSG_INTEGRATOR_FAST, vs, C, vps=vps, max_points=W * H, max_updates=16 << 20, **kw)
    if C == 256:                # label 255 is a real class here (sequence() puts it into the frames)
        cfg.dynamic_label[255] = 0
    return cfg


# name: (config keywords, sequence keywords, what happens before frame 2)
CASES = {
    "base": (dict(), dict(), None),
    "vps2": (dict(vps=2, max_blocks=1 << 16), dict(), None),
    "vps4": (dict(vps=4, max_blocks=1 << 14), dict(), None),
    "vps8": (dict(vps=8), dict(), None),
    "vps32": (dict(vps=32), dict(), None),
    "c2": (dict(C=2), dict(), None),
    "c32": (dict(C=32), dict(), None),
    "c33": (dict(C=33), dict(), None),
    "c64": (dict(C=64), dict(), None),
    "c65": (dict(C=65), dict(), None),
    "c150": (dict(vs=0.10, C=150), dict(), None),            # 10 cm: the exports of a 150- or 256-float row stay small
    "c256": (dict(vs=0.10, C=256), dict(), None),
    "colour_points": (dict(color_mode=KSG_COLOR_MODE_COLOR), dict(colours=True), None),
    "colour_probability": (dict(color_mode=KSG_COLOR_MODE_SEMANTIC_PROBABILITY), dict(), None),
    "sorted": (dict(integration_order_mode=KSG_ORDER_SORTED), dict(), None),
    "collisions0": (dict(max_consecutive_ray_collisions=0), dict(), None),
    "clear_checks3": (dict(clear_checks_every_n_frames=3), dict(), None),
    "clear_map": (dict(), dict(), "clear_map"),
    "reset": (dict(), dict(), "reset"),
    "saturated": (dict(use_const_weight=1, max_weight=1.0), dict(all_label0=True), None),
}


def log_keys(heads):
    return [tuple(b) + (int(v),) for b, v in zip(heads["block_index"].tolist(), (heads["lin_label"] & 0xFFFFFF).tolist())]


def assert_entries_equal_map(heads, pri, exp, where, rgba_tol=0):
    """Every entry's distance, weight, colours, label and log-probability row equal the voxel of the exported map, bit for bit."""
    row = {tuple(b): i for i, b in enumerate(exp["block_index"].tolist())}
    b = np.array([row[tuple(x)] for x in heads["block_index"].tolist()], np.int64)
    lin = (heads["lin_label"] & 0xFFFFFF).astype(np.int64)
    assert np.array_equal(heads["tsdf_distance"].view(np.uint32), exp["tsdf_distance"][b, lin].view(np.uint32)), where
    assert np.array_equal(heads["tsdf_weight"].view(np.uint32), exp["tsdf_weight"][b, lin].view(np.uint32)), where
    d = np.abs(heads["tsdf_rgba"].astype(np.int32) - exp["tsdf_rgba"][b, lin].astype(np.int32))
    assert d.max(initial=0) <= rgba_tol, where
    assert np.array_equal(heads["sem_rgba"], exp["sem_rgba"][b, lin]), where
    assert np.array_equal(heads["lin_label"] >> 24, exp["sem_label"][b, lin].astype(np.uint32)), where
    assert np.array_equal(pri.view(np.uint32), exp["sem_priors"][b, lin].view(np.uint32)), where


def assert_tile_order(heads, vox, vps, where):
    """What k_fast_group guarantees about the order of a frame's entries: within a tile, ascending tile-local voxel index; a tile's
    entries form at most one contiguous run per 512 of its sorted records (one slot reservation per round, which other tiles'
    reservations may split).  `vox` = the frame's update records (one per voxel update)."""
    ts = min(vps, 8)
    tps = vps // ts
    bi = heads["block_index"].astype(np.int64)
    lin = (heads["lin_label"] & 0xFFFFFF).astype(np.int64)
    loc = np.stack([lin % vps, (lin // vps) % vps, lin // (vps * vps)], axis=1)
    tile = (loc[:, 0] // ts) + tps * ((loc[:, 1] // ts) + tps * (loc[:, 2] // ts))
    v = (loc[:, 0] % ts) + ts * ((loc[:, 1] % ts) + ts * (loc[:, 2] % ts))
    key = [tuple(b) + (int(t),) for b, t in zip(bi.tolist(), tile.tolist())]
    rb, rlin = ft.block_lin(vox, vps)
    rloc = np.stack([rlin % vps, (rlin // vps) % vps, rlin // (vps * vps)], axis=1)
    rtile = (rloc[:, 0] // ts) + tps * ((rloc[:, 1] // ts) + tps * (rloc[:, 2] // ts))
    recs = {}
    for k in (tuple(b) + (int(t),) for b, t in zip(rb.tolist(), rtile.tolist())):
        recs[k] = recs.get(k, 0) + 1
    runs, last_v = {}, {}
    for i, k in enumerate(key):
        if i == 0 or key[i - 1] != k:
            runs[k] = runs.get(k, 0) + 1
        assert last_v.get(k, -1) < v[i], (where, "tile entries out of voxel order", k)
        last_v[k] = int(v[i])
    assert set(runs) == set(recs), where
    over = {k: (n, recs[k]) for k, n in runs.items() if n > -(-recs[k] // GROUP_ROUND)}
    assert not over, (where, "a tile split into more runs than slot reservations: (runs, records)", list(over.items())[:5])
    return max(runs.values(), default=0)


def check_frame(gpu, ora, cfg, kind, args, where, sg=None):
    """The frame's log against the trace of the live oracle, the device map and the oracle map.  Returns (heads, priors, records)."""
    vps = cfg.voxels_per_side
    rgba_tol = 1 if cfg.color_mode == KSG_COLOR_MODE_SEMANTIC_PROBABILITY else 0
    heads, pri = gpu.fetch_update_log()
    vox = ft.frame_records(ora, cfg, kind, args)[0]
    keys = log_keys(heads)
    assert len(set(keys)) == len(keys), f"{where}: a voxel is logged twice"
    want = ft.pairs(*ft.block_lin(vox, vps))
    got = set(keys)
    assert got == want, (where, len(got), len(want), sorted(got - want)[:5], sorted(want - got)[:5])
    assert gpu.update_log_size() == len(heads), where
    if sg is not None:
        assert sg.voxel_updates == len(vox), where
    assert_entries_equal_map(heads, pri, gpu.export(), f"{where}, device")
    assert_entries_equal_map(heads, pri, ora.export(), f"{where}, oracle", rgba_tol)
    blocks = {tuple(b) for b in gpu.last_updated_blocks().tolist()}
    assert {k[:3] for k in keys} == blocks == {tuple(b) for b in ora.last_updated_blocks().tolist()}, where
    assert_tile_order(heads, vox, vps, where)
    return heads, pri, vox


@pytest.mark.parametrize("name", list(CASES))
def test_every_frame_logs_exactly_the_traced_voxels_with_their_final_state(name):
    ckw, skw, event = CASES[name]
    cfg = fast_config(**ckw)
    gpu, ora = Integrator(cfg), OracleIntegrator(cfg)
    gpu.set_update_log(LOG)
    ft.enable(ora)
    seq = ft.sequence(W, H, cfg.num_labels, **skw)
    if name == "saturated":       # the same label-0 depth frame twice: voxels at max_weight and +truncation take unchanging updates
        seq = [seq[0], seq[0]]
    labels = set()
    for f, (kind, args) in enumerate(seq):
        if f == 2 and event == "clear_map":
            gpu.clear_map()
            ora.clear_map()
        elif f == 2 and event == "reset":
            gpu.reset()
            ora.close()
            ora = OracleIntegrator(cfg)           # ksg_reset: an empty map and fresh approximate sets
            ft.enable(ora)
        before = ora.export() if name == "saturated" else None
        sg = ft.integrate(gpu, kind, args)
        ft.integrate(ora, kind, args)
        heads, _, _ = check_frame(gpu, ora, cfg, kind, args, f"{name} frame {f} ({kind})", sg)
        assert len(heads) > 0
        labels |= set((heads["lin_label"] >> 24).tolist())
        if before is not None and f == 1:         # entries whose voxel did not change: no map diff can see them
            e = ora.export()
            assert np.array_equal(e["block_index"], before["block_index"])
            lin = (heads["lin_label"] & 0xFFFFFF).astype(np.int64)
            row = {tuple(b): i for i, b in enumerate(e["block_index"].tolist())}
            b = np.array([row[tuple(x)] for x in heads["block_index"].tolist()], np.int64)
            same = (e["tsdf_weight"][b, lin] == before["tsdf_weight"][b, lin]) & (e["tsdf_distance"][b, lin] == before["tsdf_distance"][b, lin])
            assert same.sum() > 1000, same.sum()
    if cfg.num_labels == 256:
        assert 255 in labels
    # an all-NaN depth frame: no point, no entry, and the fetch succeeds
    cam = synth.make_camera(W, H)
    nan = np.full((H, W), np.nan, np.float32)
    gpu.integrate_depth(synth.pose(0), nan, np.zeros((H, W), np.uint8), cam.K)
    heads, pri = gpu.fetch_update_log()
    assert len(heads) == 0 and pri.shape == (0, cfg.num_labels) and gpu.update_log_size() == 0
    gpu.close()
    ora.close()


def test_a_tile_of_more_than_4096_records_logs_each_voxel_once_in_reservation_runs():
    """The dense-tile scene of test_gpu_fast_voxel_items.py: one tile with more records than the shared-memory sort holds."""
    from test_gpu_fast_voxel_items import scene
    cfg, fr = scene()
    gpu, ora = Integrator(cfg), OracleIntegrator(cfg)
    gpu.set_update_log(LOG)
    ft.enable(ora)
    for f, (T, xyz, labels) in enumerate(fr):
        args = (T, xyz, labels, None)
        sg = ft.integrate(gpu, "points", args)
        ft.integrate(ora, "points", args)
        heads, _, vox = check_frame(gpu, ora, cfg, "points", args, f"dense tile frame {f}", sg)
        _, lin = ft.block_lin(vox, 16)
        cam_tile = (ft.block_lin(vox, 16)[0] == 0).all(axis=1) & ((lin % 16) < 8) & ((lin // 16 % 16) < 8) & (lin // 256 < 8)
        assert cam_tile.sum() > 4096
    gpu.close()
    ora.close()


@pytest.mark.parametrize("C", [21, 150])
def test_a_log_one_entry_too_small_reports_the_overflow_and_leaves_the_map_exact(C):
    cfg = fast_config(vs=0.05 if C == 21 else 0.10, C=C)
    seq = ft.sequence(W, H, C)
    kind, args = seq[0]
    probe = Integrator(cfg)
    probe.set_update_log(LOG)
    ft.integrate(probe, kind, args)
    roomy_heads, roomy_pri = probe.fetch_update_log()
    n0 = len(roomy_heads)
    probe.close()
    small, exact, ora = Integrator(cfg), Integrator(cfg), OracleIntegrator(cfg)
    small.set_update_log(n0 - 1)
    exact.set_update_log(n0)
    ft.enable(ora)
    for x in (small, exact, ora):
        ft.integrate(x, kind, args)
    cnt, hp, pp = ct.c_int64(123), ct.c_void_p(), ct.POINTER(ct.c_float)()
    rc = small.lib.ksg_fetch_update_log(small.handle, ct.byref(cnt), ct.byref(hp), ct.byref(pp))
    assert rc == KSG_ERR_SCRATCH_FULL and cnt.value == -1
    cnt = ct.c_int64(123)
    rc = small.lib.ksg_copy_update_log_device(small.handle, ct.byref(cnt), None, None, 0, None)
    assert rc == KSG_ERR_SCRATCH_FULL and cnt.value == -1
    a, b = small.export(), exact.export()
    assert a.keys() == b.keys() and all(np.array_equal(a[k].view(np.uint8), b[k].view(np.uint8)) for k in a)
    rep = compare_maps(a, ora.export())
    assert_parity(rep, rtol=0.0)
    assert rep["tsdf_distance_bit_mismatch"] == 0 and rep["tsdf_weight_bit_mismatch"] == 0 and rep["sem_priors_bit_mismatch"] == 0
    eh, ep = exact.fetch_update_log()

    def entries(heads, pri):
        return {k: (heads[i].tobytes(), pri[i].tobytes()) for i, k in enumerate(log_keys(heads))}
    assert len(eh) == n0 and entries(eh, ep) == entries(roomy_heads, roomy_pri)
    # the next frame, with room: a sparse subset of the points of frame 1
    T, depth, label, K = seq[1][1]
    cam = synth.make_camera(W, H)
    xyz, pix = synth.backproject(depth, cam)
    nxt = (T, np.ascontiguousarray(xyz[::40]), np.ascontiguousarray(label.reshape(-1)[pix][::40], np.uint8), None)
    sg = ft.integrate(small, "points", nxt)
    ft.integrate(ora, "points", nxt)
    heads, _, _ = check_frame(small, ora, cfg, "points", nxt, "after the overflow", sg)
    assert 0 < len(heads) < n0 - 1
    for x in (small, exact, ora):
        x.close()


@pytest.mark.parametrize("ranks,vps", [(2, 16), (3, 16), (2, 8), (3, 8)])
def test_spatial_shards_log_disjoint_owned_voxels_whose_union_is_the_unsharded_log(ranks, vps):
    C = 21
    whole = Integrator(fast_config(vps=vps))
    shards = [Integrator(fast_config(vps=vps, shard_count=ranks, shard_rank=r)) for r in range(ranks)]
    for x in [whole] + shards:
        x.set_update_log(LOG)

    def entries(heads, pri):
        keys = log_keys(heads)
        assert len(set(keys)) == len(keys)
        return {k: (heads[i].tobytes(), pri[i].tobytes()) for i, k in enumerate(keys)}

    for f, (kind, args) in enumerate(ft.sequence(W, H, C)):
        logs = []
        for x in [whole] + shards:
            ft.integrate(x, kind, args)
            logs.append(x.fetch_update_log())
        want = entries(*logs[0])
        got = {}
        for r in range(ranks):
            heads, pri = logs[r + 1]
            assert len(heads) > 0 and shards[r].update_log_size() == len(heads)
            m = owner_mask(heads["block_index"], vps, r, ranks)
            assert m[np.arange(len(heads)), heads["lin_label"] & 0xFFFFFF].all(), f"frame {f}: rank {r} logged a voxel it does not own"
            e = entries(heads, pri)
            assert not (set(e) & set(got)), f"frame {f}: ranks logged the same voxel"
            got.update(e)
        assert got == want, (f, len(got), len(want))
    for x in [whole] + shards:
        x.close()


def palette(cfg):
    return np.array([[cfg.label_color[l][k] if cfg.label_color_known[l] else 0 for k in range(4)] for l in range(256)], np.uint8)


def stack_logs(torch, logs, C):
    """Device buffers holding the logs (None = an empty delta) at a stride of more than the largest count."""
    counts = [0 if x is None else x.update_log_size() for x in logs]
    stride = max(counts) + 7
    upd = torch.zeros(len(logs) * stride * 32, dtype=torch.uint8, device="cuda")
    pri = torch.zeros(len(logs) * stride * C, dtype=torch.float32, device="cuda")
    for g, x in enumerate(logs):
        if x is not None:
            assert x.copy_update_log_device(upd[g * stride * 32:].data_ptr(), pri[g * stride * C:].data_ptr(), stride) == counts[g]
    torch.cuda.synchronize()
    return counts, stride, upd, pri


def assert_same_map(a, b, where):
    assert a.keys() == b.keys()
    for k in a:
        assert a[k].shape == b[k].shape and np.array_equal(a[k].view(np.uint8), b[k].view(np.uint8)), (where, k)


@pytest.mark.parametrize("vps,C,color_mode", [(8, 33, 1), (32, 21, 0), (4, 150, 1), (16, 256, 1)])
def test_voxel_granular_merge_off_the_default_geometry_equals_block_merge_and_the_oracle_schedule(vps, C, color_mode):
    """Four live integrators with emptied layers per batch; their logs, with an empty delta in the middle, go into ONE
    ksg_merge_voxels_device call.  It must equal ksg_merge_blocks_device of the same deltas (updated() lists included) and the numpy
    merge of the oracle's deltas (delta_merge_ref.py)."""
    import torch
    G, rounds = 4, 2
    max_blocks = {4: 1 << 14, 8: 4096, 16: 512, 32: 256}[vps]      # six integrators on one device: pools sized to the scene
    cfg = fast_config(vs=0.10 if C >= 150 else 0.05, C=C, vps=vps, color_mode=color_mode, max_blocks=max_blocks)
    pal = palette(cfg)
    by_blocks, by_voxels = Integrator(cfg), Integrator(cfg)
    gpus = [Integrator(cfg) for _ in range(G)]
    oracles = [OracleIntegrator(cfg) for _ in range(G)]
    for g in gpus:
        g.set_update_log(LOG)
    ref = dm.empty_map(vps, C)
    fr = list(frames(W, H, C, G * rounds, seed=3))
    for b in range(rounds):
        touched_b = []
        for r in range(G):
            cam, depth, label, T = fr[b * G + r]
            if C == 256:
                label = np.where(label == 1, 255, label).astype(np.uint8)
            gpus[r].clear_map()
            oracles[r].clear_map()
            gpus[r].integrate_depth(T, depth, label, cam.K)
            oracles[r].integrate_depth(T, depth, label, cam.K)
            nb, _, pool, keys = gpus[r].device_map_view()
            by_blocks.merge_blocks_device(nb, keys, pool)
            by_blocks.sync()
            touched_b.append(by_blocks.last_updated_blocks())
            ref = dm.merge(ref, oracles[r].export(), pal, cfg.max_weight, color_mode)
        counts, stride, upd, pri = stack_logs(torch, gpus[:2] + [None] + gpus[2:], C)
        assert counts[2] == 0 and min(counts[:2] + counts[3:]) > 1000
        by_voxels.merge_voxels_device(counts, stride, upd.data_ptr(), pri.data_ptr())
        got = np.unique(by_voxels.last_updated_blocks(), axis=0)
        assert np.array_equal(got, np.unique(np.concatenate(touched_b), axis=0)), b
    a = by_voxels.export()
    assert_same_map(a, by_blocks.export(), "voxel deltas / block deltas")
    rep = compare_maps(a, ref)
    assert_parity(rep, rtol=0.0)
    assert rep["tsdf_distance_bit_mismatch"] == 0 and rep["tsdf_weight_bit_mismatch"] == 0 and rep["sem_priors_bit_mismatch"] == 0, rep
    if C == 256:
        assert (a["sem_label"] == 255).any()
    for x in gpus + oracles + [by_blocks, by_voxels]:
        x.close()


def test_sixteen_voxel_granular_deltas_in_one_call_equal_sixteen_block_merges():
    import torch
    C, G = 21, 16
    cfg = fast_config(C=C, max_blocks=1024)
    by_blocks, by_voxels = Integrator(cfg), Integrator(cfg)
    gpus = [Integrator(cfg) for _ in range(G)]
    for g in gpus:
        g.set_update_log(LOG)
    touched_b = []
    for r, (cam, depth, label, T) in enumerate(frames(W, H, C, G, seed=5)):
        gpus[r].integrate_depth(T, depth, label, cam.K)
        nb, _, pool, keys = gpus[r].device_map_view()
        by_blocks.merge_blocks_device(nb, keys, pool)
        by_blocks.sync()
        touched_b.append(by_blocks.last_updated_blocks())
    counts, stride, upd, pri = stack_logs(torch, gpus, C)
    by_voxels.merge_voxels_device(counts, stride, upd.data_ptr(), pri.data_ptr())
    assert np.array_equal(np.unique(by_voxels.last_updated_blocks(), axis=0), np.unique(np.concatenate(touched_b), axis=0))
    assert_same_map(by_voxels.export(), by_blocks.export(), "16 voxel deltas / 16 block deltas")
    for x in gpus + [by_blocks, by_voxels]:
        x.close()


@pytest.mark.parametrize("vps", [8, 32])
def test_the_shim_keeps_the_host_layers_exact_after_every_fast_call(demo, tmp_path, vps):
    """shim_demo fast (eager) on each prefix of a 3-frame sequence: the host layers after k calls equal the oracle after k frames, and
    with KSG_NO_UPDATE_LOG=1 (whole-block copies) the output is byte-identical.  The shim's C is KIMERA_TOTAL_NUMBER_OF_LABELS (21)."""
    C, vs = 21, 0.05
    cfg = make_config(KSG_INTEGRATOR_FAST, vs, C, vps=vps, max_points=W * H)
    pal = np.array([[cfg.label_color[l][k] for k in range(4)] for l in range(C)], np.uint8)
    ora = OracleIntegrator(cfg)
    ora.set_color_to_label(pal[:, :3], np.arange(C, dtype=np.uint8))
    fr = []
    for cam, depth, label, T in frames(W, H, C, 3, seed=11):
        xyz, pix = synth.backproject(depth, cam)
        rgba = pal[label.reshape(-1)[pix]].copy()
        rgba[::53] = (9, 8, 7, 255)                      # unknown colour -> label 0
        fr.append((T, xyz, rgba))
    env = dict(os.environ, KSG_MAX_POINTS=str(W * H), KSG_MAX_UPDATES=str(16 << 20))
    env.pop("KSG_NO_UPDATE_LOG", None)
    for k in range(1, 4):
        ora.integrate_points(fr[k - 1][0], fr[k - 1][1], rgba=fr[k - 1][2])
        fpath = tmp_path / f"frames{k}.bin"
        write_frames(fpath, fr[:k], vs, vps, pal, [C - 1])
        outs = []
        for tag, e in (("log", env), ("blocks", dict(env, KSG_NO_UPDATE_LOG="1"))):
            opath = tmp_path / f"out{k}_{tag}.bin"
            r = subprocess.run([demo, "fast", str(fpath), str(opath)], capture_output=True, text=True, env=e, timeout=600)
            assert r.returncode == 0, r.stderr + r.stdout
            outs.append(open(opath, "rb").read())
        assert outs[0] == outs[1], f"prefix {k}: update-log sync and block copy differ"
        rep = compare_maps(read_shim_output(tmp_path / f"out{k}_log.bin", vps, C), ora.export())
        assert_parity(rep, rtol=0.0)
        assert rep["tsdf_distance_bit_mismatch"] == 0 and rep["tsdf_weight_bit_mismatch"] == 0 and rep["sem_priors_bit_mismatch"] == 0, (k, rep)
    ora.close()
