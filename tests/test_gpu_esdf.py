"""The batch ESDF of the device map (ksg_compute_esdf, csrc/ksg_esdf.cuh) equals its numpy twin (tests/esdf_ref.py) on the exported map
bit for bit in distance and flags - on integrated scenes of both integrators and on imported fields whose sites lie several unallocated
blocks from the output blocks - for any subset of outputs, in stream order behind device-side frames, and through the C++ shim in lazy
mode and its .vxblx file; plus the rejected inputs, the empty map, the untouched map and the launch count."""
import ctypes as Ct
import itertools
import os
import subprocess

import numpy as np
import pytest
import torch

from kimera_semantics_b200 import synth
from kimera_semantics_b200.capi import Integrator, KSG_INTEGRATOR_FAST, KSG_INTEGRATOR_MERGED
from parity_utils import frames, make_config
from test_shim_cpu import demo, write_frames  # noqa: F401
from test_esdf_file_cpu import esdf_words, parse_vxblx
from test_gpu_query import _same
import esdf_ref as er

pytestmark = pytest.mark.gpu
F = np.float32
W, H = 320, 240
LAUNCHES = 4


def _check(gpu, exp, vs, vps, m, min_weight=1e-4):
    got = gpu.esdf(m, min_weight=min_weight)
    want = er.esdf(exp, vs, vps, m, min_weight=min_weight)
    _same(got, want)
    return got


@pytest.mark.parametrize("itype", [KSG_INTEGRATOR_FAST, KSG_INTEGRATOR_MERGED])
def test_esdf_of_an_integrated_scene_equals_the_twin(itype):
    vs, C = 0.05, 21
    cfg = make_config(itype, vs, C, max_points=W * H, max_updates=16 << 20)
    gpu = Integrator(cfg)
    for cam, depth, label, T in frames(W, H, C, 6):
        gpu.integrate_depth(T, depth, label, cam.K)
    exp = gpu.export()
    for m in (0.4, 2.0):
        got = _check(gpu, exp, vs, cfg.voxels_per_side, m)
        fl = got["flags"]
        for bit in (er.OBSERVED, er.SURFACE) + ((er.CAPPED,) if m < 1 else ()):   # every observed voxel lies within 2 m of a site
            assert ((fl & bit) != 0).any(), (m, bit)
        assert (fl == 0).any() and not ((fl & er.CAPPED) != 0).all()
    gpu.close()


def _separated_field(vps, vs, C, seed):
    """a sphere field over a box of blocks, ~2 % unobserved voxels and one block missing, plus one far block of sites (a plane) beyond
    unallocated blocks along x and one row over in y: its sites reach the box's corner only through the x and y work sets outside the
    allocated set"""
    import mesh_ref as mr
    lo, hi = {2: (-6, 6), 8: (-2, 2), 16: (-1, 1)}[vps]
    exp = mr.sdf_export(lambda x, y, z: np.sqrt(x * x + (y - F(0.03)) ** 2 + z * z) - F(0.5), vs, vps, lo, hi)
    gap = {2: 3, 8: 2, 16: 1}[vps]                                    # 0.6, 1.6, 1.6 m of unallocated blocks along x
    far = mr.sdf_export(lambda x, y, z: x - F(0.5 * vs), vs, vps, 0, 1)          # sites: its voxel layer nearest the box
    shift = np.array([hi + gap, hi, hi - 1], np.int32)
    far["block_index"] = far["block_index"] + shift
    exp = {k: np.concatenate([exp[k], far[k]]) for k in exp}
    rng = np.random.default_rng(seed)
    nb, V = len(exp["block_index"]), vps ** 3
    exp["tsdf_weight"] = rng.choice(np.array([0.0, 0.5, 2.0], F), size=(nb, V), p=[0.01, 0.01, 0.98])
    exp["sem_priors"] = rng.uniform(-5, 0, (nb, V, C)).astype(F)
    exp["sem_rgba"] = rng.integers(0, 256, (nb, V, 4)).astype(np.uint8)
    hole = np.all(exp["block_index"] == (0, -1, 0), axis=1)
    return {k: v[~hole] for k, v in exp.items()}, shift


@pytest.mark.parametrize("vps", [2, 8, 16])
def test_esdf_of_an_imported_field_equals_the_twin(vps):
    vs, C = 0.1, 8
    exp, shift = _separated_field(vps, vs, C, vps)
    cfg = make_config(KSG_INTEGRATOR_FAST, vs, C, vps=vps, max_points=1024, max_updates=1 << 16)
    gpu = Integrator(cfg)
    gpu.import_blocks(exp)
    back = gpu.export()
    far = np.all(back["block_index"] == shift, axis=1)
    assert far.sum() == 1
    for m, mw in ((0.4, 1e-4), (1.2, 1e-4), (2.0, 1e-4), (2.0, 1.0)):
        got = _check(gpu, back, vs, vps, m, min_weight=mw)
        assert (got["flags"][far] & er.SURFACE).any()
        if m == 2.0:                                                   # the far sites change the box's output
            alone = er.esdf({k: v[~far] for k, v in back.items()}, vs, vps, m, min_weight=mw)
            assert (got["distance"][~far].view(np.uint32) != alone["distance"].view(np.uint32)).any()
    gpu.close()


def _integrated(itype=KSG_INTEGRATOR_MERGED, n=3, vs=0.05):
    cfg = make_config(itype, vs, 21, max_points=W * H, max_updates=16 << 20)
    gpu = Integrator(cfg)
    for cam, depth, label, T in frames(W, H, 21, n):
        gpu.integrate_depth(T, depth, label, cam.K)
    return gpu, cfg


def test_any_subset_of_outputs_writes_only_what_is_asked_and_leaves_the_map_alone():
    gpu, cfg = _integrated()
    vs, vps, m = 0.05, cfg.voxels_per_side, 0.6
    exp = gpu.export()
    want = er.esdf(exp, vs, vps, m)
    nb, V = len(exp["block_index"]), vps ** 3
    guard = 0xA5
    lib, h = gpu.lib, gpu.handle
    for mask in itertools.product((0, 1), repeat=3):
        bufs = {"block_index": np.full(nb * 3 * 4, guard, np.uint8), "distance": np.full(nb * V * 4, guard, np.uint8),
                "flags": np.full(nb * V, guard, np.uint8)}
        ptr = [Ct.c_void_p(b.ctypes.data) if on else None for on, b in zip(mask, bufs.values())]
        gpu.set_profiling(False)
        assert lib.ksg_compute_esdf(h, 1e-4, m, nb, *ptr) == 0
        assert gpu.get_profile()["kernel_launches"] == (LAUNCHES if (mask[1] or mask[2]) else 0), mask
        got = {"block_index": bufs["block_index"].view(np.int32).reshape(nb, 3), "distance": bufs["distance"].view(F).reshape(nb, V),
               "flags": bufs["flags"].reshape(nb, V)}
        for on, k in zip(mask, got):
            if on:
                _same(got, want, [k])
            else:
                assert (bufs[k] == guard).all(), (mask, k)
    after = gpu.export()
    for k in exp:
        assert exp[k].tobytes() == after[k].tobytes(), k
    gpu.close()


def test_rejected_and_trivial_inputs():
    gpu, cfg = _integrated(KSG_INTEGRATOR_FAST, 2)
    lib, h = gpu.lib, gpu.handle
    nb, V = gpu.num_blocks(), cfg.voxels_per_side ** 3
    dist = np.zeros(nb * V, F)

    def call(mw=1e-4, m=0.5, cap=nb, handle=h):
        return lib.ksg_compute_esdf(handle, mw, m, cap, None, Ct.c_void_p(dist.ctypes.data), None)

    bad = [dict(mw=float("nan")), dict(mw=-1.0), dict(m=0.0), dict(m=-0.5), dict(m=float("nan")), dict(m=float("inf")),
           dict(m=511 * 0.05 + 0.01), dict(cap=nb - 1), dict(cap=-1)]
    for kw in bad:
        assert call(**kw) == 1, kw
    assert lib.ksg_compute_esdf(None, 1e-4, 0.5, nb, None, None, None) == 1
    # W = ceil(m / vs) + 1 <= 512: 511 voxels is the largest max_distance accepted
    assert call(m=F(510 * 0.05)) == 0
    gpu.close()
    empty = Integrator(make_config(KSG_INTEGRATOR_FAST, 0.05, 21, max_points=1024, max_updates=1 << 16))
    empty.set_profiling(False)
    assert empty.lib.ksg_compute_esdf(empty.handle, 1e-4, 0.5, 0, None, None, None) == 0
    got = empty.esdf(0.5)
    assert got["distance"].shape == (0, 16 ** 3) and empty.get_profile()["kernel_launches"] == 0
    empty.close()
    sharded = Integrator(make_config(KSG_INTEGRATOR_FAST, 0.05, 21, max_points=1024, max_updates=1 << 16, shard_count=2, shard_rank=1))
    assert sharded.lib.ksg_compute_esdf(sharded.handle, 1e-4, 0.5, 0, None, None, None) == 1
    assert b"shard" in sharded.lib.ksg_last_error(sharded.handle)
    sharded.close()


@pytest.mark.parametrize("itype", [KSG_INTEGRATOR_FAST, KSG_INTEGRATOR_MERGED])
def test_esdf_right_after_device_frames_on_a_user_stream(itype):
    vs, C = 0.05, 21
    cfg = make_config(itype, vs, C, max_points=W * H, max_updates=16 << 20)
    gpu = Integrator(cfg)
    fr = list(frames(W, H, C, 4))
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        dev = [(torch.from_numpy(d).cuda(), torch.from_numpy(l).cuda()) for _, d, l, _ in fr]
        for (cam, _, _, Tf), (dd, dl) in zip(fr, dev):
            gpu.integrate_depth_device(Tf, dd.data_ptr(), dl.data_ptr(), W, H, cam.K, stream=st.cuda_stream)
    got = gpu.esdf(1.0)                                               # no host sync before the call
    st.synchronize()
    _same(got, er.esdf(gpu.export(), vs, cfg.voxels_per_side, 1.0))
    gpu.close()


@pytest.mark.parametrize("method", ["fast", "merged"])
def test_shim_update_esdf_batch_in_lazy_mode_equals_the_c_abi(demo, tmp_path, method):  # noqa: F811
    C, w, h, vs, m = 21, 320, 240, 0.10, 1.0
    itype = KSG_INTEGRATOR_FAST if method == "fast" else KSG_INTEGRATOR_MERGED
    cfg = make_config(itype, vs, C, max_points=w * h, max_updates=8 << 20)
    pal = np.array([[cfg.label_color[l][k] for k in range(4)] for l in range(C)], np.uint8)
    gpu = Integrator(cfg)
    gpu.set_color_to_label(pal[:, :3], np.arange(C, dtype=np.uint8))
    fr = []
    for cam, depth, label, T in frames(w, h, C, 2):
        xyz, pix = synth.backproject(depth, cam)
        rgba = pal[label.reshape(-1)[pix]].copy()
        fr.append((T, xyz, rgba))
        gpu.integrate_points(T, xyz, rgba=rgba)
    want = gpu.esdf(m)
    fpath, opath, epath = tmp_path / "frames.bin", tmp_path / "out.bin", tmp_path / "esdf.vxblx"
    write_frames(fpath, fr, vs, 16, pal, [C - 1])
    env = dict(os.environ, KSG_MAX_POINTS=str(w * h), KSG_MAX_UPDATES=str(8 << 20))
    r = subprocess.run([demo, method, str(fpath), str(opath), "lazy", "--esdf", str(m), str(epath)], capture_output=True, text=True,
                       env=env, timeout=600)
    assert r.returncode == 0, r.stderr + r.stdout
    assert "esdf:" in r.stdout and "host layers not synchronised" in r.stdout
    layer, blocks = parse_vxblx(epath)
    assert layer.type == "esdf" and layer.voxels_per_side == 16 and abs(layer.voxel_size - vs) < 1e-7
    where = {tuple(b): i for i, b in enumerate(want["block_index"].tolist())}
    assert len(blocks) == len(where)
    for b in blocks:
        i = where[tuple(round(o / (16 * vs)) for o in (b.origin_x, b.origin_y, b.origin_z))]
        dist, obs, hal, inq, fixed = esdf_words(b)
        fl = want["flags"][i]
        assert (obs == ((fl & er.OBSERVED) != 0)).all() and (fixed == ((fl & er.SURFACE) != 0)).all()
        assert not hal.any() and not inq.any()
        wd = np.where(obs, want["distance"][i], F(0))                  # unobserved: voxblox's default voxel
        assert (dist.view(np.uint32) == wd.view(np.uint32)).all()
    gpu.close()
