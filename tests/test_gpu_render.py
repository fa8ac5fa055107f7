"""Depth and semantic images of the device map (ksg_render_view / ksg_render_view_device, csrc/ksg_render.cuh) equal their numpy twin
(tests/render_ref.py) on the exported map bit for bit - every output and every flag - on integrated scenes of both integrators, on
imported fields with unobserved voxels and a missing block, in stream order behind device-side frames, for any subset of outputs, and
through the C++ shim in lazy mode; plus the rejected inputs and the launch counts."""
import ctypes as Ct
import os
import subprocess

import numpy as np
import pytest
import torch

from kimera_semantics_b200 import synth
from kimera_semantics_b200.capi import (QUERY_FIELDS, RENDER_FIELDS, Integrator, KsgError, KsgRenderOut, KSG_INTEGRATOR_FAST,
                                        KSG_INTEGRATOR_MERGED)
from parity_utils import frames, make_config
from test_shim_cpu import demo, write_frames  # noqa: F401
from test_gpu_more import read_shim_output
from test_gpu_query import _same
import mesh_ref as mr
import render_ref as rr

pytestmark = pytest.mark.gpu
F = np.float32
W, H = 320, 240


def _K(cam):
    return np.array([cam.fx, cam.fy, cam.cx, cam.cy], np.float64)


def _poses():
    """an integration pose, a novel pose between and above the stream, and one from inside the r = 2 m sphere of the synthetic world"""
    novel = synth.pose(2.5, radius=2.7, height=1.8, pitch=0.25)
    inside = np.concatenate([synth.pose(3)[:4], np.array([0.2, -0.1, 0.9], F)]).astype(F)
    return {"integrated": synth.pose(3), "novel": novel, "inside": inside}


@pytest.mark.parametrize("itype,C", [(KSG_INTEGRATOR_FAST, 21), (KSG_INTEGRATOR_MERGED, 21), (KSG_INTEGRATOR_MERGED, 150)])
def test_render_of_an_integrated_scene_equals_the_twin(itype, C):
    vs = 0.05
    cfg = make_config(itype, vs, C, max_points=W * H, max_updates=16 << 20)
    gpu = Integrator(cfg)
    for cam, depth, label, T in frames(W, H, C, 6):
        gpu.integrate_depth(T, depth, label, cam.K)
    exp = gpu.export()
    cam = synth.make_camera(W, H)
    for name, T in _poses().items():
        got = gpu.render(T, _K(cam), W, H, 0.1, 6.0)
        want = rr.render(exp, vs, cfg.voxels_per_side, T, _K(cam), W, H, 0.1, 6.0)
        _same(got, want)
        if name != "inside":                                        # from inside the sphere its surface is seen from behind: no hit
            assert (~np.isnan(got["depth"])).mean() > 0.3, name
    gpu.close()


@pytest.mark.parametrize("vps,lo,hi", [(2, -6, 6), (8, -2, 2), (16, -1, 1)])
def test_render_of_an_imported_field_equals_the_twin(vps, lo, hi):
    vs, C = 0.1, 8
    exp = mr.sdf_export(lambda x, y, z: np.sqrt(x * x + (y - F(0.03)) ** 2 + z * z) - F(0.9), vs, vps, lo, hi)
    rng = np.random.default_rng(vps)
    nb, V = len(exp["block_index"]), vps ** 3
    exp["tsdf_weight"] = rng.choice(np.array([0.0, 0.5, 2.0], F), size=(nb, V), p=[0.01, 0.01, 0.98])
    exp["sem_priors"] = rng.uniform(-5, 0, (nb, V, C)).astype(F)
    exp["sem_rgba"] = rng.integers(0, 256, (nb, V, 4)).astype(np.uint8)
    hole = np.all(exp["block_index"] == (0, -1, 0), axis=1)                # one block left out of the import
    exp = {k: v[~hole] for k, v in exp.items()}
    cfg = make_config(KSG_INTEGRATOR_FAST, vs, C, vps=vps, max_points=1024, max_updates=1 << 16)
    gpu = Integrator(cfg)
    gpu.import_blocks(exp)
    back = gpu.export()
    K = np.array([120.0, 118.0, 79.5, 59.5])
    for eye, q in (((0.1, -0.05, -1.5), (1, 0, 0, 0)), ((1.2, 0.3, -0.2), (0.7071068, 0, -0.7071068, 0))):
        T = np.array(list(q) + list(eye), F)
        got = gpu.render(T, K, 160, 120, 0.05, 4.0, min_weight=1.0)
        _same(got, rr.render(back, vs, vps, T, K, 160, 120, 0.05, 4.0, min_weight=1.0))
        assert (~np.isnan(got["depth"])).mean() > 0.2
    gpu.close()


def _device_out(n, C, guard):
    """device buffers of every output, every byte = guard"""
    def buf(nbytes):
        return torch.full((nbytes,), guard, dtype=torch.uint8, device="cuda")
    return {"depth": buf(4 * n).view(torch.float32), "points_G": buf(12 * n).view(torch.float32).view(n, 3),
            "flags": buf(n), "tsdf_distance": buf(4 * n).view(torch.float32), "tsdf_weight": buf(4 * n).view(torch.float32),
            "tsdf_rgba": buf(4 * n).view(n, 4), "sem_label": buf(n), "sem_priors": buf(4 * n * C).view(torch.float32).view(n, C),
            "sem_rgba": buf(4 * n).view(n, 4), "distance": buf(4 * n).view(torch.float32), "gradient": buf(12 * n).view(torch.float32).view(n, 3)}


def _flat(want):
    return {k: v.reshape((W * H,) + v.shape[2:]) for k, v in want.items()}


@pytest.mark.parametrize("itype", [KSG_INTEGRATOR_FAST, KSG_INTEGRATOR_MERGED])
def test_device_render_is_ordered_behind_device_frames_without_a_host_sync(itype):
    C, vs = 21, 0.05
    cfg = make_config(itype, vs, C, max_points=W * H, max_updates=16 << 20)
    gpu = Integrator(cfg)
    fr = list(frames(W, H, C, 4))
    cam = fr[0][0]
    T = synth.pose(2)
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        dev = [(torch.from_numpy(d).cuda(), torch.from_numpy(l).cuda()) for _, d, l, _ in fr]
        out = _device_out(W * H, C, 0)
        for (cam, _, _, Tf), (dd, dl) in zip(fr, dev):
            gpu.integrate_depth_device(Tf, dd.data_ptr(), dl.data_ptr(), W, H, cam.K, stream=st.cuda_stream)
        gpu.render_device(T, _K(cam), W, H, 0.1, 6.0, {k: v.data_ptr() for k, v in out.items()}, stream=st.cuda_stream)
    st.synchronize()
    got = {k: v.cpu().numpy() for k, v in out.items()}
    _same(got, _flat(rr.render(gpu.export(), vs, cfg.voxels_per_side, T, _K(cam), W, H, 0.1, 6.0)))
    gpu.close()


@pytest.mark.parametrize("wanted", [("depth",), ("points_G",), ("sem_label", "gradient"), RENDER_FIELDS])
def test_unrequested_outputs_are_never_written(wanted):
    C, vs = 21, 0.05
    cfg = make_config(KSG_INTEGRATOR_MERGED, vs, C, max_points=W * H, max_updates=16 << 20)
    gpu = Integrator(cfg)
    for cam, depth, label, Tf in frames(W, H, C, 3):
        gpu.integrate_depth(Tf, depth, label, cam.K)
    exp = gpu.export()
    T = synth.pose(1)
    guard = 0xA5
    out = _device_out(W * H, C, guard)
    torch.cuda.synchronize()
    ptrs = {k: out[k].data_ptr() for k in wanted}
    on_device = wanted
    if "points_G" not in wanted and set(wanted) & set(QUERY_FIELDS):
        # at_hit outputs without points_G: the device entry refuses them (its query reads points_G); the host entry stages the points
        with pytest.raises(KsgError):
            gpu.render_device(T, _K(cam), W, H, 0.1, 6.0, ptrs)
        on_device = ()
    else:
        gpu.render_device(T, _K(cam), W, H, 0.1, 6.0, ptrs)
    gpu.sync()
    want = _flat(rr.render(exp, vs, cfg.voxels_per_side, T, _K(cam), W, H, 0.1, 6.0))
    got = {k: v.cpu().numpy() for k, v in out.items()}
    if on_device:
        _same(got, want, on_device)
    for k in RENDER_FIELDS:
        if k not in on_device:
            assert (got[k].view(np.uint8) == guard).all(), k
    # the host entry writes exactly what it is asked for, too
    host = gpu.render(T, _K(cam), W, H, 0.1, 6.0, fields=wanted)
    assert sorted(host) == sorted(wanted)
    _same(_flat(host), want, wanted)
    gpu.close()


def test_rejected_and_trivial_inputs():
    C = 21
    cfg = make_config(KSG_INTEGRATOR_FAST, 0.05, C, max_points=1024, max_updates=1 << 16)
    gpu = Integrator(cfg)
    lib, h = gpu.lib, gpu.handle
    w, hh = 8, 6
    dep = np.zeros(w * hh, F)
    T = np.array([1, 0, 0, 0, 0, 0, 0], F)
    K = np.array([10.0, 10.0, 3.5, 2.5])
    o = KsgRenderOut(depth=dep.ctypes.data)
    fp, dp = Ct.POINTER(Ct.c_float), Ct.POINTER(Ct.c_double)

    def call(T=T, K=K, w=w, hh=hh, lo=0.1, hi=5.0, mw=1e-4, out=o, device=False):
        Tp = None if T is None else np.ascontiguousarray(T, F).ctypes.data_as(fp)
        Kp = None if K is None else np.ascontiguousarray(K, np.float64).ctypes.data_as(dp)
        op = None if out is None else Ct.byref(out)
        if device:
            return lib.ksg_render_view_device(h, Tp, Kp, w, hh, lo, hi, mw, op, None)
        return lib.ksg_render_view(h, Tp, Kp, w, hh, lo, hi, mw, op)

    assert call() == 0 and np.isnan(dep).all()                        # empty map: every pixel a miss
    bad = [dict(T=None), dict(K=None), dict(out=None), dict(T=[1, 0, 0, np.nan, 0, 0, 0]), dict(T=[1, 0, 0, 0, np.inf, 0, 0]),
           dict(K=[10.0, 10.0, np.nan, 2.5]), dict(K=[0.0, 10.0, 3.5, 2.5]), dict(K=[10.0, -1.0, 3.5, 2.5]), dict(w=0), dict(hh=-1),
           dict(lo=0.0), dict(lo=-1.0), dict(lo=float("nan")), dict(lo=float("inf"), hi=float("inf")), dict(hi=0.1), dict(hi=0.05),
           dict(hi=float("inf")), dict(hi=float("nan")), dict(mw=float("nan")), dict(mw=-1.0),
           # the step rule: (0.05 / 4) / r_max >= max_depth * 2^-20 holds up to max_depth ~ 1.2e4 m here, and not at 1e5 m
           dict(hi=1.0e5), dict(K=[1e-3, 1e-3, 3.5, 2.5], hi=50.0)]
    for kw in bad:
        assert call(**kw) == 1, kw
        assert call(device=True, **kw) == 1, kw
    assert lib.ksg_render_view(None, T.ctypes.data_as(fp), K.ctypes.data_as(dp), w, hh, 0.1, 5.0, 1e-4, Ct.byref(o)) == 1
    assert call(hi=1.0e4) == 0
    # the device entry needs points_G for an at_hit output; the host entry stages it
    fl = np.zeros(w * hh, np.uint8)
    only_hit = KsgRenderOut.of({"flags": fl.ctypes.data})
    assert call(out=only_hit) == 0
    assert call(out=only_hit, device=True) == 1
    # launches: nothing wanted 0, depth / points alone 1, any at_hit output 2
    d = {k: torch.zeros(3 * w * hh, device="cuda") for k in ("depth", "points_G", "distance")}
    torch.cuda.synchronize()
    gpu.set_profiling(False)                                          # zeroes the launch counter
    assert call(out=KsgRenderOut()) == 0 and call(out=KsgRenderOut(), device=True) == 0
    assert gpu.get_profile()["kernel_launches"] == 0
    gpu.render_device(T, K, w, hh, 0.1, 5.0, {"depth": d["depth"].data_ptr()})
    gpu.sync()
    assert gpu.get_profile()["kernel_launches"] == 1
    gpu.render_device(T, K, w, hh, 0.1, 5.0, {"points_G": d["points_G"].data_ptr()})
    gpu.sync()
    assert gpu.get_profile()["kernel_launches"] == 2
    gpu.render_device(T, K, w, hh, 0.1, 5.0, {k: v.data_ptr() for k, v in d.items()})
    gpu.sync()
    assert gpu.get_profile()["kernel_launches"] == 4
    gpu.close()
    sharded = Integrator(make_config(KSG_INTEGRATOR_FAST, 0.05, C, max_points=1024, max_updates=1 << 16, shard_count=2, shard_rank=1))
    assert sharded.lib.ksg_render_view(sharded.handle, T.ctypes.data_as(fp), K.ctypes.data_as(dp), w, hh, 0.1, 5.0, 1e-4, Ct.byref(o)) == 1
    assert b"shard" in sharded.lib.ksg_last_error(sharded.handle)
    assert sharded.lib.ksg_render_view_device(sharded.handle, T.ctypes.data_as(fp), K.ctypes.data_as(dp), w, hh, 0.1, 5.0, 1e-4,
                                              Ct.byref(o), None) == 1
    sharded.close()


@pytest.mark.parametrize("method", ["fast", "merged"])
def test_shim_render_in_lazy_mode_equals_the_c_abi(demo, tmp_path, method):
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
    cam = synth.make_camera(w, h)
    T, K = synth.pose(1), _K(cam)
    want = gpu.render(T, K, w, h, 0.1, 6.0)
    fpath, opath, rin, rout = tmp_path / "frames.bin", tmp_path / "out.bin", tmp_path / "pose.bin", tmp_path / "r.bin"
    write_frames(fpath, fr, vs, 16, pal, [C - 1])
    with open(rin, "wb") as f:
        f.write(T.astype(F).tobytes())
        f.write(K.tobytes())
        f.write(np.array([w, h], np.int32).tobytes())
        f.write(np.array([0.1, 6.0, 1e-4], F).tobytes())
    env = dict(os.environ, KSG_MAX_POINTS=str(w * h), KSG_MAX_UPDATES=str(8 << 20))
    r = subprocess.run([demo, method, str(fpath), str(opath), "lazy", "--render", str(rin), str(rout)], capture_output=True, text=True,
                       env=env, timeout=600)
    assert r.returncode == 0, r.stderr + r.stdout
    assert "host layers not synchronised" in r.stdout
    _same(read_shim_output(opath, 16, C), exp)                      # the shim integrated the same map
    raw, n, off, got = open(rout, "rb").read(), w * h, 0, {}
    for k, dt, per in (("depth", F, 1), ("points_G", F, 3), ("flags", np.uint8, 1), ("tsdf_distance", F, 1), ("tsdf_weight", F, 1),
                       ("tsdf_rgba", np.uint8, 4), ("sem_label", np.uint8, 1), ("sem_priors", F, C), ("sem_rgba", np.uint8, 4),
                       ("distance", F, 1), ("gradient", F, 3)):
        a = np.frombuffer(raw, dt, n * per, off)
        off += a.nbytes
        got[k] = a.reshape(want[k].shape)
    assert off == len(raw)
    _same(got, want)
    assert (~np.isnan(got["depth"])).mean() > 0.3
    gpu.close()
