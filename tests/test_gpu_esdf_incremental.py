"""The device ESDF layer (ksg_update_esdf / ksg_export_esdf / ksg_query_esdf[_device], csrc/ksg_esdf.cuh): after every update it equals
the batch entry ksg_compute_esdf bit for bit, and its stats equal the numpy model of the incremental rule (tests/esdf_incremental_ref.py)
- over `fast` and `merged` streams updated after every frame and after every third, after imports, block and voxel merges, clear_map,
reset and a parameter change.  An update with nothing changed launches nothing, changed_only lists exactly the rewritten blocks, device
frames on a user stream need no host sync, the inputs the batch entry rejects are rejected, and the point queries equal their twin on the
exported layer bit for bit (blocks allocated after the update answer as unallocated, unwanted outputs stay untouched, the device entry
runs in stream order).  Last, the C++ shim's incremental host layer equals its batch layer, in lazy and eager mode and in its .vxblx file."""
import ctypes as Ct
import os
import subprocess

import numpy as np
import pytest
import torch

from kimera_semantics_b200 import synth
from kimera_semantics_b200.capi import ESDF_QUERY_FIELDS, Integrator, KsgEsdfQueryOut, KSG_INTEGRATOR_FAST, KSG_INTEGRATOR_MERGED
from parity_utils import frames, make_config
from test_shim_cpu import demo, write_frames  # noqa: F401
from test_esdf_file_cpu import esdf_words, parse_vxblx
from test_gpu_query import _same, _mixed_points
import esdf_incremental_ref as ir

pytestmark = pytest.mark.gpu
F = np.float32
W, H, VS, C = 320, 240, 0.05, 21


def _keys(a):
    return {tuple(int(c) for c in b) for b in np.asarray(a).reshape(-1, 3)}


class Checked:
    """an integrator with the model beside it: update() checks the layer against ksg_compute_esdf and the stats against the model"""

    def __init__(self, cfg):
        self.gpu, self.cfg, self.state, self.changed = Integrator(cfg), cfg, None, set()

    def touched(self):
        self.changed |= _keys(self.gpu.last_updated_blocks())

    def update(self, m, mw=1e-4, full=None):
        st = self.gpu.update_esdf(m, min_weight=mw)
        exp = self.gpu.export()
        self.state, want_st = ir.update(self.state, exp, self.changed, VS, self.cfg.voxels_per_side, m, min_weight=mw)
        if full is not None:
            want_st["full"] = int(full)          # the model cannot see clear / reset / import: the caller says what it expects
            if full:
                self.state, want_st = ir.update(None, exp, [], VS, self.cfg.voxels_per_side, m, min_weight=mw)
        self.changed = set()
        assert st == want_st, (st, want_st)
        layer = self.gpu.export_esdf()
        _same(layer, self.gpu.esdf(m, min_weight=mw))
        part = self.gpu.export_esdf(changed_only=True)
        assert _keys(part["block_index"]) == self.state["D"]
        at = {tuple(b): i for i, b in enumerate(layer["block_index"].tolist())}
        rows = [at[tuple(b)] for b in part["block_index"].tolist()]
        assert part["block_index"].tolist() == sorted(part["block_index"].tolist(), key=lambda b: (b[2], b[1], b[0]))
        _same(part, {"block_index": layer["block_index"][rows], "distance": layer["distance"][rows], "flags": layer["flags"][rows]})
        return st, layer


@pytest.mark.parametrize("every", [1, 3])
@pytest.mark.parametrize("itype", [KSG_INTEGRATOR_FAST, KSG_INTEGRATOR_MERGED])
def test_updates_along_a_stream_equal_the_batch_entry_and_the_model(itype, every):
    cfg = make_config(itype, VS, C, max_points=W * H, max_updates=16 << 20)
    c = Checked(cfg)
    stats = []
    for k, (cam, depth, label, T) in enumerate(frames(W, H, C, 12)):
        c.gpu.integrate_depth(T, depth, label, cam.K)
        c.touched()
        if k % every == every - 1:
            stats.append(c.update(1.0)[0])
    assert stats[0]["full"] == 1 and all(s["full"] == 0 for s in stats[1:])
    assert any(s["site_changed"] > 0 for s in stats[1:])
    assert all(s["z_blocks"] <= s["blocks"] for s in stats)     # the camera sweeps this small room: D is often the whole map
    c.gpu.close()


def test_map_edits_clear_reset_and_new_parameters():
    cfg = make_config(KSG_INTEGRATOR_FAST, VS, C, max_points=W * H, max_updates=16 << 20)
    c = Checked(cfg)
    fr = list(frames(W, H, C, 8))
    for cam, depth, label, T in fr[:2]:
        c.gpu.integrate_depth(T, depth, label, cam.K)
    c.update(1.0, full=True)
    # import: overwrite the map's blocks with noise and add far blocks; the import does not stamp, so the next update is full
    exp = c.gpu.export()
    rng = np.random.default_rng(5)
    exp["tsdf_distance"] = (exp["tsdf_distance"] + rng.normal(0, VS, exp["tsdf_distance"].shape)).astype(F)
    far = {k: v[:2].copy() for k, v in exp.items()}
    far["block_index"] = far["block_index"] + np.array([40, 0, 0], np.int32)
    c.gpu.import_blocks({k: np.concatenate([exp[k], far[k]]) for k in exp})
    c.update(1.0, full=True)
    # block merges and voxel merges stamp the blocks they write: incremental
    d = Integrator(cfg)
    d.set_update_log(1 << 20)
    d.integrate_depth(fr[2][3], fr[2][1], fr[2][2], fr[2][0].K)
    nb, _, pool, keys = d.device_map_view()
    c.gpu.merge_blocks_device(nb, keys, pool)
    c.gpu.sync()
    c.touched()
    st = c.update(1.0, full=False)[0]
    assert st["changed_blocks"] > 0 and st["z_blocks"] <= st["blocks"] - 2          # the two far blocks lie beyond Rb of every edit
    n = d.update_log_size()
    upd = torch.zeros(n * 32, dtype=torch.uint8, device="cuda")
    pri = torch.zeros(n * C, dtype=torch.float32, device="cuda")
    assert d.copy_update_log_device(upd.data_ptr(), pri.data_ptr(), n) == n
    torch.cuda.synchronize()
    c.gpu.merge_voxels_device([n], n, upd.data_ptr(), pri.data_ptr())
    c.gpu.sync()
    c.touched()
    c.update(1.0, full=False)
    d.close()
    # new parameters: full; the same again: nothing changed, no launch
    c.update(0.6, full=True)
    c.update(0.6, mw=0.5, full=True)
    c.gpu.set_profiling(False)
    st = c.gpu.update_esdf(0.6, min_weight=0.5)
    assert st["changed_blocks"] == 0 and st["z_blocks"] == 0 and c.gpu.get_profile()["kernel_launches"] == 0
    # clear_map (the stamps restart while frame_stamp does not) and reset: the layer is dropped until the next update, which is full
    for edit in ("clear_map", "reset"):
        getattr(c.gpu, edit)()
        assert c.gpu.lib.ksg_export_esdf(c.gpu.handle, 0, 0, None, None, None, None) == 1
        c.changed = set()
        for cam, depth, label, T in fr[3:5]:
            c.gpu.integrate_depth(T, depth, label, cam.K)
        c.update(1.0, full=True)
        cam, depth, label, T = fr[5]
        c.gpu.integrate_depth(T, depth, label, cam.K)
        c.touched()
        c.update(1.0, full=False)
    c.gpu.close()


def test_no_change_no_launch_and_device_frames_without_a_host_sync():
    cfg = make_config(KSG_INTEGRATOR_MERGED, VS, C, max_points=W * H, max_updates=16 << 20)
    gpu = Integrator(cfg)
    fr = list(frames(W, H, C, 5))
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        dev = [(torch.from_numpy(d).cuda(), torch.from_numpy(l).cuda()) for _, d, l, _ in fr]
        for (cam, _, _, Tf), (dd, dl) in zip(fr[:3], dev):
            gpu.integrate_depth_device(Tf, dd.data_ptr(), dl.data_ptr(), W, H, cam.K, stream=st.cuda_stream)
    gpu.update_esdf(1.0)                                                # no host sync before the call
    _same(gpu.export_esdf(), gpu.esdf(1.0))
    gpu.set_profiling(False)
    s = gpu.update_esdf(1.0)
    assert s["changed_blocks"] == 0 and s["site_blocks"] == 0 and gpu.get_profile()["kernel_launches"] == 0
    with torch.cuda.stream(st):
        for (cam, _, _, Tf), (dd, dl) in zip(fr[3:], dev[3:]):
            gpu.integrate_depth_device(Tf, dd.data_ptr(), dl.data_ptr(), W, H, cam.K, stream=st.cuda_stream)
    s = gpu.update_esdf(1.0)
    assert s["full"] == 0 and s["changed_blocks"] > 0
    before = gpu.export_esdf()
    _same(before, gpu.esdf(1.0))
    # the batch entry at other parameters reads and writes none of the layer's state: the next update has nothing to do
    gpu.esdf(0.6, min_weight=0.5)
    gpu.set_profiling(False)
    s = gpu.update_esdf(1.0)
    assert s["full"] == 0 and s["changed_blocks"] == 0 and gpu.get_profile()["kernel_launches"] == 0
    after = gpu.export_esdf()
    assert after.keys() == before.keys() and all(after[k].tobytes() == before[k].tobytes() for k in before)
    gpu.close()


def test_rejected_inputs():
    cfg = make_config(KSG_INTEGRATOR_FAST, VS, C, max_points=W * H, max_updates=16 << 20)
    gpu = Integrator(cfg)
    lib, h = gpu.lib, gpu.handle
    cam, depth, label, T = next(iter(frames(W, H, C, 1)))
    gpu.integrate_depth(T, depth, label, cam.K)
    p = np.zeros((4, 3), F)
    out = np.zeros(4, F)
    q = KsgEsdfQueryOut(distance=out.ctypes.data)
    n = Ct.c_int64()
    assert lib.ksg_export_esdf(h, 0, 0, Ct.byref(n), None, None, None) == 1          # before any update
    assert lib.ksg_query_esdf(h, 4, p.ctypes.data, Ct.byref(q)) == 1
    assert lib.ksg_query_esdf_device(h, 0, None, Ct.byref(q), None) == 1
    for mw, m in ((float("nan"), 0.5), (-1.0, 0.5), (1e-4, 0.0), (1e-4, -0.5), (1e-4, float("nan")), (1e-4, float("inf")),
                  (1e-4, 511 * VS + 0.01)):
        assert lib.ksg_update_esdf(h, mw, m, None) == 1, (mw, m)
        assert lib.ksg_export_esdf(h, 0, 0, Ct.byref(n), None, None, None) == 1     # a rejected call creates no layer
    assert lib.ksg_update_esdf(None, 1e-4, 0.5, None) == 1
    assert lib.ksg_update_esdf(h, 1e-4, F(510 * VS), None) == 0                      # W = 512
    assert lib.ksg_export_esdf(h, 0, 0, Ct.byref(n), None, None, None) == 0 and n.value == gpu.num_blocks()
    nb, V = n.value, cfg.voxels_per_side ** 3
    d = np.zeros(nb * V, F)
    assert lib.ksg_export_esdf(h, 0, nb - 1, Ct.byref(n), None, d.ctypes.data, None) == 1
    assert lib.ksg_query_esdf(h, -1, p.ctypes.data, Ct.byref(q)) == 1
    assert lib.ksg_query_esdf(h, 4, None, Ct.byref(q)) == 1
    assert lib.ksg_query_esdf(h, 4, p.ctypes.data, None) == 1
    assert lib.ksg_query_esdf(h, 4, p.ctypes.data, Ct.byref(q)) == 0
    gpu.close()
    sharded = Integrator(make_config(KSG_INTEGRATOR_FAST, VS, C, max_points=1024, max_updates=1 << 16, shard_count=2, shard_rank=1))
    assert sharded.lib.ksg_update_esdf(sharded.handle, 1e-4, 0.5, None) == 1
    assert b"shard" in sharded.lib.ksg_last_error(sharded.handle)
    sharded.close()


@pytest.mark.parametrize("itype", [KSG_INTEGRATOR_FAST, KSG_INTEGRATOR_MERGED])
def test_queries_equal_the_twin_on_the_exported_layer(itype):
    cfg = make_config(itype, VS, C, max_points=W * H, max_updates=16 << 20)
    gpu = Integrator(cfg)
    vps = cfg.voxels_per_side
    fr = list(frames(W, H, C, 6))
    for cam, depth, label, T in fr[:4]:
        gpu.integrate_depth(T, depth, label, cam.K)
    gpu.update_esdf(1.0)
    layer = gpu.export_esdf()
    pts = _mixed_points(gpu.export(), VS, vps, 3000, 1)
    want = ir.esdf_query(layer, VS, vps, pts)
    assert ((want["flags"] & 8) != 0).sum() > 500 and ((want["voxel_flags"] & 4) != 0).any()
    _same(gpu.query_esdf(pts), want)
    # frames after the update: new blocks answer as unallocated, the layer's blocks as before
    for cam, depth, label, T in fr[4:]:
        gpu.integrate_depth(T, depth, label, cam.K)
    new = _keys(gpu.export()["block_index"]) - _keys(layer["block_index"])
    assert new
    b = np.array(sorted(new), np.float64)
    inside = ((b + 0.5) * vps * VS).astype(F)
    got = gpu.query_esdf(np.concatenate([pts, inside]))
    _same({k: v[: len(pts)] for k, v in got.items()}, want)
    assert (got["flags"][len(pts):] == 0).all() and np.isnan(got["voxel_distance"][len(pts):]).all()
    # unwanted outputs are never written; the device entry, in stream order, and the host entry with the same subset of outputs
    n = len(pts)
    guard = 0xA5
    dp = torch.from_numpy(pts).cuda()
    sizes = {"flags": n, "voxel_flags": n, "voxel_distance": 4 * n, "distance": 4 * n, "gradient": 12 * n}
    for keep in (("flags",), ("voxel_distance", "gradient"), ESDF_QUERY_FIELDS):
        bufs = {k: torch.full((sizes[k],), guard, dtype=torch.uint8, device="cuda") for k in ESDF_QUERY_FIELDS}
        host = {k: np.full(sizes[k], guard, np.uint8) for k in ESDF_QUERY_FIELDS}
        st = torch.cuda.Stream()
        st.wait_stream(torch.cuda.current_stream())
        gpu.query_esdf_device(dp.data_ptr(), n, {k: bufs[k].data_ptr() for k in keep}, stream=st.cuda_stream)
        st.synchronize()
        q = KsgEsdfQueryOut(**{k: host[k].ctypes.data for k in keep})
        assert gpu.lib.ksg_query_esdf(gpu.handle, n, pts.ctypes.data, Ct.byref(q)) == 0
        for raws in ({k: v.cpu().numpy() for k, v in bufs.items()}, host):
            for k in ESDF_QUERY_FIELDS:
                raw = raws[k]
                if k not in keep:
                    assert (raw == guard).all(), k
                    continue
                dt = np.float32 if k in ("voxel_distance", "distance", "gradient") else np.uint8
                v = raw.view(dt).reshape(want[k].shape)
                _same({k: v}, {k: want[k]})
    gpu.close()


@pytest.mark.parametrize("mode", ["lazy", "eager"])
def test_shim_update_esdf_equals_its_batch_layer(demo, tmp_path, mode):  # noqa: F811
    """shim_demo --esdf-every 2: SemanticTsdfServer::updateEsdf after every second frame into one host layer, then the batch layer of the
    same map; both files and the C-ABI's batch ESDF agree"""
    w, h, vs, m = 320, 240, 0.10, 1.0
    cfg = make_config(KSG_INTEGRATOR_FAST, vs, C, max_points=w * h, max_updates=8 << 20)
    pal = np.array([[cfg.label_color[l][k] for k in range(4)] for l in range(C)], np.uint8)
    gpu = Integrator(cfg)
    gpu.set_color_to_label(pal[:, :3], np.arange(C, dtype=np.uint8))
    fr = []
    for cam, depth, label, T in frames(w, h, C, 5):
        xyz, pix = synth.backproject(depth, cam)
        rgba = pal[label.reshape(-1)[pix]].copy()
        fr.append((T, xyz, rgba))
        gpu.integrate_points(T, xyz, rgba=rgba)
    want = gpu.esdf(m)
    fpath, opath, ipath, bpath = tmp_path / "frames.bin", tmp_path / "out.bin", tmp_path / "inc.vxblx", tmp_path / "batch.vxblx"
    write_frames(fpath, fr, vs, 16, pal, [C - 1])
    env = dict(os.environ, KSG_MAX_POINTS=str(w * h), KSG_MAX_UPDATES=str(8 << 20))
    r = subprocess.run([demo, "fast", str(fpath), str(opath), mode, "--esdf-every", "2", str(m), str(ipath), "--esdf", str(m), str(bpath)],
                       capture_output=True, text=True, env=env, timeout=600)
    assert r.returncode == 0, r.stderr + r.stdout
    assert "esdf-every: 3 updates" in r.stdout
    inc, bat = parse_vxblx(ipath), parse_vxblx(bpath)
    assert inc[0].type == bat[0].type == "esdf" and len(inc[1]) == len(bat[1]) == len(want["block_index"])
    by_origin = lambda blocks: {(b.origin_x, b.origin_y, b.origin_z): esdf_words(b) for b in blocks}   # noqa: E731
    a, b = by_origin(inc[1]), by_origin(bat[1])
    assert a.keys() == b.keys()
    for o in a:
        for x, y in zip(a[o], b[o]):
            assert np.asarray(x).tobytes() == np.asarray(y).tobytes(), o
    gpu.close()
