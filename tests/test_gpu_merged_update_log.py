"""The update log of the `merged` integrator (ksg_set_update_log / ksg_fetch_update_log, k_merged_log_heads / k_merged_log_write in
ksg_log.cuh): one entry per voxel the frame updated, with the voxel's final state, in record order.

Every comparison is bit for bit.  The voxels a frame updated come from the oracle (merged_update_trace.py, checked on the CPU by
test_merged_update_trace_cpu.py); every entry's state must equal both the device export and the oracle export."""
import ctypes as ct
import json
import os
import subprocess
import sys

import numpy as np
import pytest

import merged_update_trace as tr
from kimera_semantics_b200 import synth
from kimera_semantics_b200.capi import (Integrator, KSG_BUNDLE_ORDER_CANONICAL, KSG_BUNDLE_ORDER_LIBSTDCXX, KSG_INTEGRATOR_MERGED,
                                        owner_mask)
from oracle.oracle_py import OracleIntegrator
from parity_utils import assert_parity, compare_maps, frames, make_config
from test_gpu_more import read_shim_output
from test_shim_cpu import demo, write_frames  # noqa: F401

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
KSG_ERR_SCRATCH_FULL = 4


def log_pairs(heads):
    return tr.pairs(heads["block_index"], heads["lin_label"] & 0xFFFFFF)


def assert_log_equals_map(heads, pri, exp, where):
    """Every entry's distance, weight, colours, label and log-probability row equal the voxel of the exported map, bit for bit."""
    row = {tuple(b): i for i, b in enumerate(exp["block_index"].tolist())}
    b = np.array([row[tuple(x)] for x in heads["block_index"].tolist()], np.int64)
    lin = (heads["lin_label"] & 0xFFFFFF).astype(np.int64)
    assert np.array_equal(heads["tsdf_distance"].view(np.uint32), exp["tsdf_distance"][b, lin].view(np.uint32)), where
    assert np.array_equal(heads["tsdf_weight"].view(np.uint32), exp["tsdf_weight"][b, lin].view(np.uint32)), where
    assert np.array_equal(heads["tsdf_rgba"], exp["tsdf_rgba"][b, lin]), where
    assert np.array_equal(heads["sem_rgba"], exp["sem_rgba"][b, lin]), where
    assert np.array_equal(heads["lin_label"] >> 24, exp["sem_label"][b, lin].astype(np.uint32)), where
    assert np.array_equal(pri.view(np.uint32), exp["sem_priors"][b, lin].view(np.uint32)), where


def assert_same_map(a, b, where=""):
    assert a.keys() == b.keys()
    for k in a:
        assert a[k].shape == b[k].shape and np.array_equal(a[k].view(np.uint8), b[k].view(np.uint8)), (where, k)


def sequence(W, H, C, n=2, seed=0):
    """(kind, args) frames: n depth frames, then the points of one more frame integrated as freespace points."""
    out = []
    for cam, depth, label, T in frames(W, H, C, n + 1, seed=seed):
        out.append(("depth", (T, depth, label, cam.K)))
    T, depth, label, cam = out[-1][1][0], out[-1][1][1], out[-1][1][2], synth.make_camera(W, H)
    xyz, pix = synth.backproject(depth, cam)
    out[-1] = ("freespace", (T, xyz, label.reshape(-1)[pix].astype(np.uint8)))
    return out


def integrate(x, kind, args):
    if kind == "depth":
        return x.integrate_depth(*args)
    T, xyz, labels = args
    return x.integrate_points(T, xyz, labels=labels, freespace=(kind == "freespace"))


def traced(cfg, kind, args):
    if kind == "depth":
        T, depth, _label, K = args
        return tr.pairs(*tr.updated_voxels_depth(cfg, T, depth, K))
    T, xyz, _labels = args
    return tr.pairs(*tr.updated_voxels_points(cfg, T, xyz, freespace=(kind == "freespace")))


CASES = [  # (voxel size, C, anti-grazing, bundle order)
    (0.05, 21, 0, KSG_BUNDLE_ORDER_CANONICAL), (0.05, 21, 0, KSG_BUNDLE_ORDER_LIBSTDCXX), (0.05, 21, 1, KSG_BUNDLE_ORDER_CANONICAL),
    (0.02, 21, 0, KSG_BUNDLE_ORDER_CANONICAL), (0.02, 21, 1, KSG_BUNDLE_ORDER_LIBSTDCXX),
    (0.05, 33, 0, KSG_BUNDLE_ORDER_CANONICAL), (0.05, 64, 1, KSG_BUNDLE_ORDER_CANONICAL),
]


@pytest.mark.parametrize("vs,C,ag,order", CASES)
def test_every_frame_logs_exactly_the_updated_voxels_with_their_final_state(vs, C, ag, order):
    W, H = 160, 120
    cfg = make_config(KSG_INTEGRATOR_MERGED, vs, C, max_points=W * H, max_updates=16 << 20, enable_anti_grazing=ag, merged_bundle_order=order)
    gpu, ora = Integrator(cfg), OracleIntegrator(cfg)
    gpu.set_update_log(1 << 22)
    for f, (kind, args) in enumerate(sequence(W, H, C)):
        sg = integrate(gpu, kind, args)
        integrate(ora, kind, args)
        heads, pri = gpu.fetch_update_log()
        got, want = log_pairs(heads), traced(cfg, kind, args)
        assert len(got) == len(heads), f"frame {f}: duplicate entries"
        assert got == want, (f, len(got), len(want), len(got - want), len(want - got))
        assert 0 < len(heads) <= sg.voxel_updates
        assert gpu.update_log_size() == len(heads)
        g, o = gpu.export(), ora.export()
        assert_log_equals_map(heads, pri, g, f"frame {f}, device")
        assert_log_equals_map(heads, pri, o, f"frame {f}, oracle")
        blocks = {tuple(b) for b in gpu.last_updated_blocks().tolist()}
        assert {p[:3] for p in got} == blocks
        keys = [tuple(b) for b in heads["block_index"].tolist()]      # the entries of one block are contiguous
        assert sum(1 for i in range(1, len(keys)) if keys[i] != keys[i - 1]) == len(blocks) - 1
        zyx = [(k[2], k[1], k[0]) for k in keys]                       # blocks in index order: z, then y, then x
        assert zyx == sorted(zyx)
    gpu.close()
    ora.close()


@pytest.fixture(scope="module")
def route_report():
    from gpu_merged_log_check import ENV_VARIANTS
    env = {k: v for k, v in os.environ.items() if k not in ENV_VARIANTS}
    r = subprocess.run([sys.executable, os.path.join(HERE, "gpu_merged_log_check.py")], capture_output=True, text=True, timeout=900, env=env)
    assert r.returncode == 0, r.stderr[-2000:]
    line = [l for l in r.stdout.splitlines() if l.startswith("REPORT ")][-1]
    return json.loads(line[len("REPORT "):])


def test_the_log_is_the_same_bytes_under_every_apply_route_and_on_every_run(route_report):
    """The scenes with hot voxels and segments on the route thresholds: the log bytes under KSG_MERGED_TILE_APPLY=1,
    KSG_LONG_LEN=4096, apply_mode 1 and hot_voxel_mode 1 / 2, and from a second integrator, equal those of the default routes;
    frame 0 logs the traced voxels with the exported state."""
    from gpu_merged_log_check import CFG_VARIANTS, ENV_VARIANTS, SCENES
    assert set(route_report) == set(SCENES)
    for name, r in route_report.items():
        assert not r["failures"], (name, r["failures"])
        base = r["runs"]["default"]
        assert all(f[0] > 0 for f in base), name
        assert all(f[4] for v in r["runs"].values() for f in v), (name, "log entries differ from the exported map")
        configs = {"default", "default_again"} | {f"{k}={v}" for k, v in ENV_VARIANTS.items()}
        configs |= {k for k in CFG_VARIANTS if not (k.startswith("hot_voxel") and name.endswith("_c33"))}
        assert set(r["runs"]) == configs, name
        bad = {k: [(f, v[f][3] != base[f][3]) for f in range(len(v)) if v[f] != base[f]] for k, v in r["runs"].items() if v != base}
        assert not bad, (name, "configuration: [(frame, the exported map differs too)]", bad)


def test_an_empty_cloud_logs_nothing_and_the_log_off_launches_what_it_always_did():
    W, H, C = 160, 120, 21
    cfg = make_config(KSG_INTEGRATOR_MERGED, 0.05, C, max_points=W * H, max_updates=16 << 20)
    on, off, ora = Integrator(cfg), Integrator(cfg), OracleIntegrator(cfg)
    on.set_update_log(1 << 20)
    fr = list(frames(W, H, C, 3))
    for cam, depth, label, T in fr[:2]:
        on.integrate_depth(T, depth, label, cam.K)
        off.integrate_depth(T, depth, label, cam.K)
        ora.integrate_depth(T, depth, label, cam.K)
    assert on.update_log_size() > 0
    on.integrate_points(fr[1][3], np.zeros((0, 3), np.float32))
    off.integrate_points(fr[1][3], np.zeros((0, 3), np.float32))
    assert on.update_log_size() == 0 and len(on.fetch_update_log()[0]) == 0
    # every point closer than min_ray_length_m: a frame with points but no update record
    on.integrate_points(fr[1][3], np.full((10, 3), 1e-3, np.float32))
    off.integrate_points(fr[1][3], np.full((10, 3), 1e-3, np.float32))
    assert on.update_log_size() == 0
    pa, pb = on.get_profile(), off.get_profile()
    # per frame with entries: k_merged_log_heads, k_merged_log_keys, k_merged_log_write; DeviceSelect::Flagged, DeviceRadixSort::SortPairs
    assert pa["kernel_launches"] - pb["kernel_launches"] == 2 * 3 and pa["library_calls"] - pb["library_calls"] == 2 * 2
    on.set_update_log(0)
    cam, depth, label, T = fr[2]
    for x in (on, off, ora):
        x.integrate_depth(T, depth, label, cam.K)
    pa2, pb2 = on.get_profile(), off.get_profile()
    assert pa2["kernel_launches"] - pa["kernel_launches"] == pb2["kernel_launches"] - pb["kernel_launches"]
    assert pa2["library_calls"] - pa["library_calls"] == pb2["library_calls"] - pb["library_calls"]
    a, b = on.export(), off.export()
    assert_same_map(a, b, "log on / off")
    assert_parity(compare_maps(a, ora.export()), rtol=0.0)
    for x in (on, off, ora):
        x.close()


def test_a_log_one_entry_too_small_reports_the_overflow_and_leaves_the_map_exact():
    W, H, C = 160, 120, 21
    cfg = make_config(KSG_INTEGRATOR_MERGED, 0.05, C, max_points=W * H, max_updates=16 << 20)
    fr = list(frames(W, H, C, 2))
    probe = Integrator(cfg)
    probe.set_update_log(1 << 20)
    cam, depth, label, T = fr[0]
    probe.integrate_depth(T, depth, label, cam.K)
    full_heads, full_pri = probe.fetch_update_log()
    n0 = len(full_heads)
    probe.close()
    small, exact, ora = Integrator(cfg), Integrator(cfg), OracleIntegrator(cfg)
    small.set_update_log(n0 - 1)
    exact.set_update_log(n0)
    for x in (small, exact, ora):
        x.integrate_depth(T, depth, label, cam.K)
    cnt, hp, pp = ct.c_int64(123), ct.c_void_p(), ct.POINTER(ct.c_float)()
    rc = small.lib.ksg_fetch_update_log(small.handle, ct.byref(cnt), ct.byref(hp), ct.byref(pp))
    assert rc == KSG_ERR_SCRATCH_FULL and cnt.value == -1
    cnt = ct.c_int64(123)
    rc = small.lib.ksg_copy_update_log_device(small.handle, ct.byref(cnt), None, None, 0, None)
    assert rc == KSG_ERR_SCRATCH_FULL and cnt.value == -1
    assert_same_map(small.export(), exact.export(), "overflowed log")
    assert_parity(compare_maps(small.export(), ora.export()), rtol=0.0)
    eh, ep = exact.fetch_update_log()
    assert eh.tobytes() == full_heads.tobytes() and ep.tobytes() == full_pri.tobytes()
    # the next frame with room: a sparse subset of frame 1's points
    cam, depth, label, T = fr[1]
    xyz, pix = synth.backproject(depth, cam)
    xyz, lab = np.ascontiguousarray(xyz[::40]), label.reshape(-1)[pix][::40].astype(np.uint8)
    for x in (small, ora):
        x.integrate_points(T, xyz, labels=lab)
    heads, pri = small.fetch_update_log()
    assert 0 < len(heads) < n0 - 1
    assert log_pairs(heads) == tr.pairs(*tr.updated_voxels_points(cfg, T, xyz))
    o = ora.export()
    assert_parity(compare_maps(small.export(), o), rtol=0.0)
    assert_log_equals_map(heads, pri, o, "after the overflow")
    for x in (small, exact, ora):
        x.close()


def test_spatial_shards_log_disjoint_owned_voxels_whose_union_is_the_unsharded_log():
    W, H, C = 160, 120, 21
    base = dict(max_points=W * H, max_updates=16 << 20)
    whole = Integrator(make_config(KSG_INTEGRATOR_MERGED, 0.05, C, **base))
    ranks = [Integrator(make_config(KSG_INTEGRATOR_MERGED, 0.05, C, shard_count=2, shard_rank=r, **base)) for r in range(2)]
    for x in [whole] + ranks:
        x.set_update_log(1 << 20)

    def entries(heads, pri):
        keys = [tuple(b) + (int(v),) for b, v in zip(heads["block_index"].tolist(), (heads["lin_label"] & 0xFFFFFF).tolist())]
        return {k: (heads[i].tobytes(), pri[i].tobytes()) for i, k in enumerate(keys)} if len(set(keys)) == len(keys) else None

    for cam, depth, label, T in frames(W, H, C, 3):
        logs = []
        for x in [whole] + ranks:
            x.integrate_depth(T, depth, label, cam.K)
            logs.append(x.fetch_update_log())
        want = entries(*logs[0])
        got = {}
        for r in range(2):
            heads, pri = logs[r + 1]
            assert len(heads) > 0
            m = owner_mask(heads["block_index"], 16, r, 2)
            assert m[np.arange(len(heads)), heads["lin_label"] & 0xFFFFFF].all(), f"rank {r} logged a voxel it does not own"
            e = entries(heads, pri)
            assert e is not None and not (set(e) & set(got))
            got.update(e)
        assert want is not None and got == want
    for x in [whole] + ranks:
        x.close()


def test_merged_voxel_granular_deltas_merge_to_the_same_map_as_whole_block_deltas():
    """The `merged` twin of test_gpu_delta_merge.py::test_voxel_granular_deltas_merge_to_the_same_map_as_whole_block_deltas: live
    integrators whose layers are emptied (ksg_clear_map) before each frame, their update logs stacked and merged with one
    ksg_merge_voxels_device call per batch, against ksg_merge_blocks_device of the same deltas, bit for bit, updated() lists included."""
    import torch
    W, H, C, G, rounds = 320, 240, 21, 3, 2
    cfg = make_config(KSG_INTEGRATOR_MERGED, 0.05, C, max_points=W * H, max_updates=16 << 20)
    by_blocks, by_voxels = Integrator(cfg), Integrator(cfg)
    gpus = [Integrator(cfg) for _ in range(G)]
    for g in gpus:
        g.set_update_log(1 << 20)
    fr = list(frames(W, H, C, G * rounds))
    for b in range(rounds):
        sizes = []
        for r in range(G):
            cam, depth, label, T = fr[b * G + r]
            gpus[r].clear_map()
            gpus[r].integrate_depth(T, depth, label, cam.K)
            sizes.append(gpus[r].update_log_size())
        assert min(sizes) > 1000
        stride = max(sizes) + 5
        upd = torch.zeros(G * stride * 32, dtype=torch.uint8, device="cuda")
        pri = torch.zeros(G * stride * C, dtype=torch.float32, device="cuda")
        for r in range(G):
            n = gpus[r].copy_update_log_device(upd[r * stride * 32:].data_ptr(), pri[r * stride * C:].data_ptr(), stride)
            assert n == sizes[r]
        torch.cuda.synchronize()
        by_voxels.merge_voxels_device(sizes, stride, upd.data_ptr(), pri.data_ptr())
        touched_v = by_voxels.last_updated_blocks()
        touched_b = []
        for r in range(G):
            nb, _, pool, keys = gpus[r].device_map_view()
            by_blocks.merge_blocks_device(nb, keys, pool)
            by_blocks.sync()
            touched_b.append(by_blocks.last_updated_blocks())
        assert np.array_equal(np.unique(touched_v, axis=0), np.unique(np.concatenate(touched_b), axis=0))
        for r in range(G):   # the merges ran frames of their own on the merging integrators; the deltas' logs are unchanged
            assert gpus[r].update_log_size() == sizes[r]
    assert_same_map(by_voxels.export(), by_blocks.export(), "voxel deltas / block deltas")
    for x in gpus + [by_blocks, by_voxels]:
        x.close()


def test_the_shim_keeps_the_host_layers_exact_after_every_merged_call(demo, tmp_path):
    """shim_demo merged (eager) on each prefix of a 3-frame sequence: the host layers after k calls equal the oracle after k frames;
    with KSG_NO_UPDATE_LOG=1 (whole-block copies) the output is byte-identical."""
    C, w, h, vs = 21, 320, 240, 0.05
    cfg = make_config(KSG_INTEGRATOR_MERGED, vs, C, max_points=w * h)
    pal = np.array([[cfg.label_color[l][k] for k in range(4)] for l in range(C)], np.uint8)
    ora = OracleIntegrator(cfg)
    ora.set_color_to_label(pal[:, :3], np.arange(C, dtype=np.uint8))
    fr = []
    for cam, depth, label, T in frames(w, h, C, 3):
        xyz, pix = synth.backproject(depth, cam)
        rgba = pal[label.reshape(-1)[pix]].copy()
        rgba[::53] = (9, 8, 7, 255)                      # unknown colour -> label 0
        fr.append((T, xyz, rgba))
    env = dict(os.environ, KSG_MAX_POINTS=str(w * h), KSG_MAX_UPDATES=str(16 << 20))
    env.pop("KSG_NO_UPDATE_LOG", None)
    for k in range(1, 4):
        ora.integrate_points(fr[k - 1][0], fr[k - 1][1], rgba=fr[k - 1][2])
        fpath = tmp_path / f"frames{k}.bin"
        write_frames(fpath, fr[:k], vs, 16, pal, [C - 1])
        outs = []
        for tag, e in (("log", env), ("blocks", dict(env, KSG_NO_UPDATE_LOG="1"))):
            opath = tmp_path / f"out{k}_{tag}.bin"
            r = subprocess.run([demo, "merged", str(fpath), str(opath)], capture_output=True, text=True, env=e, timeout=600)
            assert r.returncode == 0, r.stderr + r.stdout
            outs.append(open(opath, "rb").read())
        assert outs[0] == outs[1], f"prefix {k}: update-log sync and block copy differ"
        rep = compare_maps(read_shim_output(tmp_path / f"out{k}_log.bin", 16, C), ora.export())
        assert_parity(rep, rtol=0.0)
        assert rep["tsdf_distance_bit_mismatch"] == 0 and rep["tsdf_weight_bit_mismatch"] == 0 and rep["sem_priors_bit_mismatch"] == 0, (k, rep)
    ora.close()
