"""Point queries on the device map (ksg_query_points / ksg_query_points_device, csrc/ksg_query.cuh) equal their numpy twin
(tests/query_ref.py) on the exported map bit for bit - every output field and every flag, on integrated scenes of both integrators, on
imported fields whose stencils straddle blocks, in stream order behind device-side frames, for any subset of outputs, and through the C++
shim in lazy mode."""
import ctypes as Ct
import os
import subprocess

import numpy as np
import pytest
import torch

from kimera_semantics_b200 import synth
from kimera_semantics_b200.capi import QUERY_FIELDS, Integrator, KsgQueryOut, KSG_INTEGRATOR_FAST, KSG_INTEGRATOR_MERGED
from parity_utils import frames, make_config
from test_shim_cpu import demo, write_frames  # noqa: F401
from test_gpu_more import read_shim_output
import mesh_ref as mr
import query_ref as qr

pytestmark = pytest.mark.gpu
F = np.float32


def _same(got, want, keys=None):
    for k in keys or want:
        a, b = np.asarray(got[k]), np.asarray(want[k])
        assert a.shape == b.shape, k
        if a.dtype == np.float32:
            bad = a.view(np.uint32) != b.view(np.uint32)
        else:
            bad = a != b
        assert not bad.any(), f"{k}: {int(bad.sum())} mismatches, first at {np.argwhere(bad)[:3].tolist()}"


def _mixed_points(exp, vs, vps, n, seed):
    """uniform over the map's bounding box, near the surface, on voxel faces and centres, in unallocated space, NaN / inf / far out"""
    rng = np.random.default_rng(seed)
    bi = exp["block_index"].astype(np.float64)
    lo, hi = bi.min(axis=0) * vps * vs, (bi.max(axis=0) + 1) * vps * vs
    uni = rng.uniform(lo, hi, (n, 3))
    V = vps ** 3
    lin = np.arange(V)
    sel = np.argwhere((exp["tsdf_weight"] > 0) & (np.abs(exp["tsdf_distance"]) < 2 * vs))
    sel = sel[rng.integers(0, len(sel), n)]
    g = bi[sel[:, 0]].astype(np.int64) * vps + np.stack([lin % vps, (lin // vps) % vps, lin // (vps * vps)], 1)[sel[:, 1]]
    near = (g + 0.5) * vs + rng.uniform(-2 * vs, 2 * vs, (n, 3))
    face = (g[: n // 4] + rng.integers(0, 2, (n // 4, 3))).astype(F) * F(vs)          # corners / faces of observed voxels
    centre = (g[n // 4: n // 2].astype(F) + F(0.5)) * F(vs)
    edge = face.copy()
    edge[:, 1] = ((g[: n // 4, 1] + 0.5) * vs)                                          # on a face in x and z only
    empty = hi + rng.uniform(1.0, 5.0, (64, 3))
    bad = np.array([[np.nan, 0, 0], [0, np.inf, 0], [0, 0, -np.inf], [1e12, 0, 0], [0, -3e8, 0], [np.nan] * 3], np.float64)
    return np.concatenate([uni, near, face, centre, edge, empty, bad]).astype(F)


def _integrated(itype, C, n_frames=6, W=320, H=240, vs=0.05):
    cfg = make_config(itype, vs, C, max_points=W * H, max_updates=16 << 20)
    gpu = Integrator(cfg)
    for cam, depth, label, T in frames(W, H, C, n_frames):
        gpu.integrate_depth(T, depth, label, cam.K)
    return gpu, cfg


@pytest.mark.parametrize("itype,C", [(KSG_INTEGRATOR_FAST, 21), (KSG_INTEGRATOR_MERGED, 21), (KSG_INTEGRATOR_MERGED, 150)])
def test_queries_on_an_integrated_scene_equal_the_twin(itype, C):
    gpu, cfg = _integrated(itype, C)
    exp = gpu.export()
    vs, vps = cfg.voxel_size, cfg.voxels_per_side
    p = _mixed_points(exp, vs, vps, 20000, seed=C + itype)
    got = gpu.query_points(p)
    want = qr.query(exp, vs, vps, p)
    _same(got, want)
    fl = got["flags"]
    for bit in (qr.ALLOCATED, qr.OBSERVED, qr.INTERPOLATED, qr.GRADIENT):
        assert ((fl & bit) != 0).any() and not ((fl & bit) != 0).all(), bit       # every case occurs
    assert (fl[-6:] == 0).all()
    # another min_weight moves the observed set; the twin follows
    got = gpu.query_points(p, min_weight=5.0, priors=False)
    want = qr.query({k: v for k, v in exp.items() if k != "sem_priors"}, vs, vps, p, min_weight=5.0)
    _same(got, want)
    gpu.close()


@pytest.mark.parametrize("itype", [KSG_INTEGRATOR_FAST, KSG_INTEGRATOR_MERGED])
def test_device_query_is_ordered_behind_device_frames_without_a_host_sync(itype):
    W, H, C, vs = 320, 240, 21, 0.05
    cfg = make_config(itype, vs, C, max_points=W * H, max_updates=16 << 20)
    gpu = Integrator(cfg)
    fr = list(frames(W, H, C, 4))
    cam, depth, label, T = fr[0]
    gpu.integrate_depth(T, depth, label, cam.K)                       # a map to pick the query points from
    p = _mixed_points(gpu.export(), vs, cfg.voxels_per_side, 8000, seed=7)
    n = len(p)
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        d_p = torch.from_numpy(p).cuda()
        dev = [(torch.from_numpy(d).cuda(), torch.from_numpy(l).cuda()) for _, d, l, _ in fr[1:]]
        out = {"flags": torch.empty(n, dtype=torch.uint8, device="cuda"), "tsdf_distance": torch.empty(n, device="cuda"),
               "tsdf_weight": torch.empty(n, device="cuda"), "tsdf_rgba": torch.empty((n, 4), dtype=torch.uint8, device="cuda"),
               "sem_label": torch.empty(n, dtype=torch.uint8, device="cuda"), "sem_priors": torch.empty((n, C), device="cuda"),
               "sem_rgba": torch.empty((n, 4), dtype=torch.uint8, device="cuda"), "distance": torch.empty(n, device="cuda"),
               "gradient": torch.empty((n, 3), device="cuda")}
        for (cam, _, _, T), (dd, dl) in zip(fr[1:], dev):
            gpu.integrate_depth_device(T, dd.data_ptr(), dl.data_ptr(), W, H, cam.K, stream=st.cuda_stream)
        gpu.query_points_device(d_p.data_ptr(), n, {k: v.data_ptr() for k, v in out.items()}, stream=st.cuda_stream)
    st.synchronize()
    got = {k: v.cpu().numpy() for k, v in out.items()}
    _same(got, qr.query(gpu.export(), vs, cfg.voxels_per_side, p))
    gpu.close()


@pytest.mark.parametrize("vps,lo,hi", [(2, -3, 3), (8, -2, 2), (16, -1, 1)])
def test_stencils_across_blocks_of_an_imported_field(vps, lo, hi):
    vs, C = 0.1, 8
    exp = mr.sdf_export(lambda x, y, z: np.sqrt(x * x + (y - F(0.03)) ** 2 + z * z) - F(0.37), vs, vps, lo, hi)
    rng = np.random.default_rng(vps)
    nb, V = len(exp["block_index"]), vps ** 3
    exp["tsdf_weight"] = rng.choice(np.array([0.0, 0.5, 2.0], F), size=(nb, V), p=[0.004, 0.004, 0.992])
    exp["sem_priors"] = rng.uniform(-5, 0, (nb, V, C)).astype(F)
    exp["sem_rgba"] = rng.integers(0, 256, (nb, V, 4)).astype(np.uint8)
    hole = np.all(exp["block_index"] == (0, -1, 0), axis=1)                # one block left out of the import
    exp = {k: v[~hole] for k, v in exp.items()}
    cfg = make_config(KSG_INTEGRATOR_FAST, vs, C, vps=vps, max_points=1024, max_updates=1 << 16)
    gpu = Integrator(cfg)
    gpu.import_blocks(exp)
    back = gpu.export()
    # points within 1.5 voxels of block corners (8 blocks), edges (4) and faces (2)
    bs = vps * vs
    n = 6000
    corner = rng.integers(lo + 1, hi, (n, 3)) * bs
    p = rng.uniform(lo * bs, hi * bs, (n, 3))
    near = rng.uniform(-1.5 * vs, 1.5 * vs, (n, 3))
    k = np.arange(n) % 3                                                     # 0: corner, 1: edge, 2: face
    for a in range(3):
        on = a < 3 - k
        p[on, a] = corner[on, a] + near[on, a]
    p = p.astype(F)
    got = gpu.query_points(p, min_weight=1.0)
    _same(got, qr.query(back, vs, vps, p, min_weight=1.0))
    assert ((got["flags"] & qr.GRADIENT) != 0).mean() > 0.2
    assert ((got["flags"] & qr.ALLOCATED) == 0).any()
    gpu.close()


def _device_out(n, C, guard):
    """device buffers of every output, every byte = guard"""
    def buf(nbytes):
        return torch.full((nbytes,), guard, dtype=torch.uint8, device="cuda")
    return {"flags": buf(n), "tsdf_distance": buf(4 * n).view(torch.float32), "tsdf_weight": buf(4 * n).view(torch.float32),
            "tsdf_rgba": buf(4 * n).view(n, 4), "sem_label": buf(n), "sem_priors": buf(4 * n * C).view(torch.float32).view(n, C),
            "sem_rgba": buf(4 * n).view(n, 4), "distance": buf(4 * n).view(torch.float32), "gradient": buf(12 * n).view(torch.float32).view(n, 3)}


@pytest.mark.parametrize("wanted", [("flags",), ("sem_priors",), QUERY_FIELDS])
def test_unrequested_outputs_are_never_written(wanted):
    gpu, cfg = _integrated(KSG_INTEGRATOR_MERGED, 21, n_frames=3)
    exp = gpu.export()
    p = _mixed_points(exp, cfg.voxel_size, cfg.voxels_per_side, 4000, seed=11)
    n, C = len(p), cfg.num_labels
    guard = 0xA5
    out = _device_out(n, C, guard)
    host = {k: v.cpu().numpy() for k, v in out.items()}                  # host arrays of the same shapes, every byte = guard
    d_p = torch.from_numpy(p).cuda()
    torch.cuda.synchronize()
    gpu.query_points_device(d_p.data_ptr(), n, {k: out[k].data_ptr() for k in wanted})
    gpu.sync()
    # the host entry with the same subset of outputs
    q = KsgQueryOut(**{k: host[k].ctypes.data for k in wanted})
    assert gpu.lib.ksg_query_points(gpu.handle, n, p.ctypes.data, 1e-4, Ct.byref(q)) == 0
    want = qr.query(exp, cfg.voxel_size, cfg.voxels_per_side, p)
    for got in ({k: v.cpu().numpy() for k, v in out.items()}, host):
        _same(got, want, wanted)
        for k in QUERY_FIELDS:
            if k not in wanted:
                assert (got[k].view(np.uint8) == guard).all(), k
    gpu.close()


def test_rejected_and_trivial_inputs():
    C = 21
    cfg = make_config(KSG_INTEGRATOR_FAST, 0.05, C, max_points=1024, max_updates=1 << 16)
    gpu = Integrator(cfg)
    p = np.zeros((4, 3), F)
    fl = np.zeros(4, np.uint8)
    q = KsgQueryOut(flags=fl.ctypes.data)
    lib, h = gpu.lib, gpu.handle
    assert lib.ksg_query_points(h, 4, p.ctypes.data, 1e-4, Ct.byref(q)) == 0
    assert lib.ksg_query_points(h, -1, p.ctypes.data, 1e-4, Ct.byref(q)) == 1
    assert lib.ksg_query_points(h, 4, p.ctypes.data, float("nan"), Ct.byref(q)) == 1
    assert lib.ksg_query_points(h, 4, p.ctypes.data, -1.0, Ct.byref(q)) == 1
    assert lib.ksg_query_points(h, 4, None, 1e-4, Ct.byref(q)) == 1
    assert lib.ksg_query_points(h, 4, p.ctypes.data, 1e-4, None) == 1
    assert lib.ksg_query_points(None, 4, p.ctypes.data, 1e-4, Ct.byref(q)) == 1
    assert lib.ksg_query_points_device(h, -1, None, 1e-4, Ct.byref(q), None) == 1
    assert lib.ksg_query_points_device(h, 4, None, float("nan"), Ct.byref(q), None) == 1
    assert lib.ksg_query_points(h, 0, None, 1e-4, Ct.byref(q)) == 0
    assert lib.ksg_query_points_device(h, 0, None, 1e-4, Ct.byref(q), None) == 0
    assert (fl == 0).all()                                          # empty map: nothing allocated
    # n > 0 with NULL points is refused even when no output is wanted (the kernel would read them)
    none = KsgQueryOut()
    assert lib.ksg_query_points(h, 4, None, 1e-4, Ct.byref(none)) == 1
    assert lib.ksg_query_points_device(h, 4, None, 1e-4, Ct.byref(none), None) == 1
    # no output wanted: OK without a launch; one wanted output: one launch
    d_p = torch.from_numpy(p).cuda()
    torch.cuda.synchronize()
    gpu.set_profiling(False)                                        # zeroes the launch counter
    assert lib.ksg_query_points(h, 4, p.ctypes.data, 1e-4, Ct.byref(none)) == 0
    assert lib.ksg_query_points_device(h, 4, d_p.data_ptr(), 1e-4, Ct.byref(none), None) == 0
    assert gpu.get_profile()["kernel_launches"] == 0
    gpu.query_points_device(d_p.data_ptr(), 4, {"flags": torch.zeros(4, dtype=torch.uint8, device="cuda").data_ptr()})
    gpu.sync()
    assert gpu.get_profile()["kernel_launches"] == 1
    gpu.close()
    sharded = Integrator(make_config(KSG_INTEGRATOR_FAST, 0.05, C, max_points=1024, max_updates=1 << 16, shard_count=2, shard_rank=1))
    assert sharded.lib.ksg_query_points(sharded.handle, 4, p.ctypes.data, 1e-4, Ct.byref(q)) == 1
    assert b"shard" in sharded.lib.ksg_last_error(sharded.handle)
    assert sharded.lib.ksg_query_points_device(sharded.handle, 4, p.ctypes.data, 1e-4, Ct.byref(q), None) == 1
    sharded.close()


@pytest.mark.parametrize("method", ["fast", "merged"])
def test_shim_queries_in_lazy_mode_equal_the_c_abi(demo, tmp_path, method):
    C, w, h, vs = 21, 320, 240, 0.10
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
    exp = gpu.export()
    p = _mixed_points(exp, vs, 16, 5000, seed=3)
    want = gpu.query_points(p)
    fpath, opath, qin, qout = tmp_path / "frames.bin", tmp_path / "out.bin", tmp_path / "q.bin", tmp_path / "r.bin"
    write_frames(fpath, fr, vs, 16, pal, [C - 1])
    with open(qin, "wb") as f:
        f.write(np.int32(len(p)).tobytes())
        f.write(p.tobytes())
    env = dict(os.environ, KSG_MAX_POINTS=str(w * h), KSG_MAX_UPDATES=str(8 << 20))
    r = subprocess.run([demo, method, str(fpath), str(opath), "lazy", "--query", str(qin), str(qout)], capture_output=True, text=True,
                       env=env, timeout=600)
    assert r.returncode == 0, r.stderr + r.stdout
    assert "host layers not synchronised" in r.stdout
    _same(read_shim_output(opath, 16, C), exp)                      # the shim integrated the same map
    raw, n, off, got = open(qout, "rb").read(), len(p), 0, {}
    for k, dt, per in (("flags", np.uint8, 1), ("tsdf_distance", F, 1), ("tsdf_weight", F, 1), ("tsdf_rgba", np.uint8, 4),
                       ("sem_label", np.uint8, 1), ("sem_priors", F, C), ("sem_rgba", np.uint8, 4), ("distance", F, 1), ("gradient", F, 3)):
        a = np.frombuffer(raw, dt, n * per, off)
        off += a.nbytes
        got[k] = a.reshape(want[k].shape)
    assert off == len(raw)
    _same(got, want)
    gpu.close()
