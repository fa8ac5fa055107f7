"""The device mesh layer (ksg_update_mesh / ksg_export_mesh / ksg_mesh_view_device, csrc/ksg_mesh.cuh): after every update it equals the
batch entry ksg_extract_mesh bit for bit, its stats equal the model of the dirty-set rule (tests/mesh_incremental_ref.py), and
changed_only lists exactly R - over `fast` and `merged` streams updated after every frame and after every third, after imports, block
and voxel merges (including one voxel merge that reaches only the diagonal lower neighbour), clear_map, reset and a new min_weight.  An
unchanged map launches nothing, the view equals the export once reordered by key, the rejected inputs are rejected, and the C++ shim's
updateMesh results assemble into its final mesh and its .ply file."""
import ctypes as Ct
import os
import subprocess

import numpy as np
import pytest
import torch

from kimera_semantics_b200 import synth
from kimera_semantics_b200.capi import Integrator, KsgMeshStats, KSG_INTEGRATOR_FAST, KSG_INTEGRATOR_MERGED
from parity_utils import frames, make_config
from test_shim_cpu import demo, write_frames  # noqa: F401
from test_ply_cpu import parse_ply
import mesh_incremental_ref as ir

pytestmark = pytest.mark.gpu
F = np.float32
W, H, VS, C = 320, 240, 0.05, 21
MESH_KEYS = ("vertices", "rgba", "labels", "block_index", "block_first")


def _keys(a):
    return {tuple(int(c) for c in b) for b in np.asarray(a).reshape(-1, 3)}


def _same(a, b):
    for k in MESH_KEYS:
        assert a[k].shape == b[k].shape and a[k].tobytes() == b[k].tobytes(), k


def _rows(mesh, blocks):
    """the extract_mesh-layout dict of `blocks` (in that order) out of `mesh`"""
    at = {tuple(b): i for i, b in enumerate(mesh["block_index"].tolist())}
    f = mesh["block_first"]
    idx = [at[tuple(b)] for b in blocks]
    pick = lambda k: np.concatenate([mesh[k][f[i]:f[i + 1]] for i in idx]) if idx else mesh[k][:0]   # noqa: E731
    first = np.concatenate([[0], np.cumsum([f[i + 1] - f[i] for i in idx])]).astype(np.int64)
    return {"vertices": pick("vertices"), "rgba": pick("rgba"), "labels": pick("labels"),
            "block_index": np.array(blocks, np.int32).reshape(-1, 3), "block_first": first}


class Checked:
    """an integrator with the model beside it: update() checks the layer against ksg_extract_mesh and the stats against the model"""

    def __init__(self, cfg):
        self.gpu, self.cfg, self.prev, self.mw, self.changed = Integrator(cfg), cfg, None, None, set()

    def touched(self):
        self.changed |= _keys(self.gpu.last_updated_blocks())

    def update(self, mw=1e-4, full=None):
        st = self.gpu.update_mesh(mw)
        batch = self.gpu.extract_mesh(mw)
        keys = _keys(batch["block_index"])
        is_full = self.prev is None or mw != self.mw if full is None else full   # the model cannot see clear / reset / import
        if not is_full and not self.changed and keys == self.prev:
            Cs, R = set(), set()
        else:
            Cs, R = ir.dirty_sets(keys, None if is_full else self.prev, self.changed)
        counts = {tuple(b): int(batch["block_first"][i + 1] - batch["block_first"][i]) for i, b in enumerate(batch["block_index"].tolist())}
        want = dict(blocks=len(keys), full=int(is_full), changed_blocks=len(Cs), remeshed_blocks=len(R),
                    vertices=int(batch["block_first"][-1]), remeshed_vertices=sum(counts[b] for b in R))
        assert st == want, (st, want)
        self.prev, self.mw, self.changed = keys, mw, set()
        layer = self.gpu.export_mesh()
        _same(layer, batch)
        part = self.gpu.export_mesh(changed_only=True)
        order = sorted(R, key=lambda b: (b[2], b[1], b[0]))
        assert part["block_index"].tolist() == [list(b) for b in order]
        _same(part, _rows(layer, order))
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
            stats.append(c.update()[0])
    assert stats[0]["full"] == 1 and all(s["full"] == 0 for s in stats[1:])
    assert any(0 < s["remeshed_blocks"] < s["blocks"] for s in stats[1:])
    assert all(s["remeshed_vertices"] <= s["vertices"] for s in stats)
    c.gpu.close()


def _voxel_entry(block, lin, dist, wgt, label, n_labels):
    rec = np.zeros(1, dtype=[("b", "<i4", 3), ("lin_label", "<u4"), ("dist", "<f4"), ("wgt", "<f4"), ("rgba", "<u4"), ("srgba", "<u4")])
    rec["b"] = block
    rec["lin_label"] = lin | (label << 24)
    rec["dist"], rec["wgt"], rec["rgba"], rec["srgba"] = dist, wgt, 0xFF0000FF, 0xFF00FF00
    return torch.from_numpy(rec.view(np.uint8).copy()).cuda(), torch.zeros(n_labels, dtype=torch.float32, device="cuda")


def test_map_edits_clear_reset_and_new_min_weight():
    cfg = make_config(KSG_INTEGRATOR_FAST, VS, C, max_points=W * H, max_updates=16 << 20)
    vps = cfg.voxels_per_side
    c = Checked(cfg)
    fr = list(frames(W, H, C, 8))
    for cam, depth, label, T in fr[:2]:
        c.gpu.integrate_depth(T, depth, label, cam.K)
    c.update(full=True)
    # import: overwrite the map's blocks with noise and add far-away blocks; the import does not stamp, so the next update is full
    exp = c.gpu.export()
    rng = np.random.default_rng(5)
    exp["tsdf_distance"] = (exp["tsdf_distance"] + rng.normal(0, VS, exp["tsdf_distance"].shape)).astype(F)
    far = {k: v[:2].copy() for k, v in exp.items()}
    far["block_index"] = far["block_index"] + np.array([40, 0, 0], np.int32)
    c.gpu.import_blocks({k: np.concatenate([exp[k], far[k]]) for k in exp})
    c.update(full=True)
    # block merges and voxel merges stamp the blocks they write: incremental
    d = Integrator(cfg)
    d.set_update_log(1 << 20)
    d.integrate_depth(fr[2][3], fr[2][1], fr[2][2], fr[2][0].K)
    nb, _, pool, keys = d.device_map_view()
    c.gpu.merge_blocks_device(nb, keys, pool)
    c.gpu.sync()
    c.touched()
    st = c.update(full=False)[0]
    assert 0 < st["remeshed_blocks"] < st["blocks"]
    n = d.update_log_size()
    upd = torch.zeros(n * 32, dtype=torch.uint8, device="cuda")
    pri = torch.zeros(n * C, dtype=torch.float32, device="cuda")
    assert d.copy_update_log_device(upd.data_ptr(), pri.data_ptr(), n) == n
    torch.cuda.synchronize()
    c.gpu.merge_voxels_device([n], n, upd.data_ptr(), pri.data_ptr())
    c.gpu.sync()
    c.touched()
    c.update(full=False)
    d.close()
    # the diagonal case: one voxel merge that flips only voxel (0, 0, 0) of block B, a cube corner of B - (1, 1, 1) and of no face
    # neighbour's cube in that block's corner; B - (1, 1, 1) must be re-meshed, and its mesh changes
    exp = c.gpu.export()
    at = {tuple(b): i for i, b in enumerate(exp["block_index"].tolist())}
    lin = lambda x, y, z: x + vps * (y + vps * z)                                                   # noqa: E731
    target = None
    for b, i in at.items():
        lo = (b[0] - 1, b[1] - 1, b[2] - 1)
        corners = [((lo[0] + ox, lo[1] + oy, lo[2] + oz), lin(0 if ox else vps - 1, 0 if oy else vps - 1, 0 if oz else vps - 1))
                   for oz in (0, 1) for oy in (0, 1) for ox in (0, 1)]
        if all(k in at and exp["tsdf_weight"][at[k], v] > 1e-3 for k, v in corners):
            target = (b, lo)
            break
    assert target is not None
    b, lo = target
    before = _rows(c.gpu.export_mesh(), [lo])
    d0 = float(exp["tsdf_distance"][at[b], 0])
    w0 = float(exp["tsdf_weight"][at[b], 0])
    upd, pri = _voxel_entry(b, 0, -d0 if d0 != 0 else -VS, 1000.0 * w0, 3, C)
    torch.cuda.synchronize()
    c.gpu.merge_voxels_device([1], 1, upd.data_ptr(), pri.data_ptr())
    c.gpu.sync()
    c.touched()
    assert c.changed == {b}
    e2 = c.gpu.export()
    assert np.sign(e2["tsdf_distance"][at[b], 0]) != np.sign(d0)
    st, layer = c.update(full=False)
    assert st["changed_blocks"] == 1 and 1 < st["remeshed_blocks"] <= 8
    after = _rows(layer, [lo])
    assert before["vertices"].tobytes() != after["vertices"].tobytes()
    # a new min_weight: full; the same again: nothing changed, no launch
    c.update(mw=0.5, full=True)
    c.gpu.set_profiling(False)
    st = c.gpu.update_mesh(0.5)
    assert st["changed_blocks"] == 0 and st["remeshed_blocks"] == 0 and c.gpu.get_profile()["kernel_launches"] == 0
    # clear_map (the stamps restart while frame_stamp does not) and reset: the layer is dropped until the next update, which is full
    for edit in ("clear_map", "reset"):
        getattr(c.gpu, edit)()
        n = Ct.c_int64()
        assert c.gpu.lib.ksg_export_mesh(c.gpu.handle, 0, 0, None, None, None, 0, None, None, Ct.byref(n), Ct.byref(n)) == 1
        assert c.gpu.lib.ksg_mesh_view_device(c.gpu.handle, Ct.byref(n), Ct.byref(n), None, None, None, None, None) == 1
        c.changed = set()
        for cam, depth, label, T in fr[3:5]:
            c.gpu.integrate_depth(T, depth, label, cam.K)
        c.update(mw=0.5, full=True)
        cam, depth, label, T = fr[5]
        c.gpu.integrate_depth(T, depth, label, cam.K)
        c.touched()
        c.update(mw=0.5, full=False)
    c.gpu.close()


@pytest.mark.parametrize("itype", [KSG_INTEGRATOR_FAST, KSG_INTEGRATOR_MERGED])
def test_view_equals_the_export(itype):
    cfg = make_config(itype, VS, C, max_points=W * H, max_updates=16 << 20)
    gpu = Integrator(cfg)
    for k, (cam, depth, label, T) in enumerate(frames(W, H, C, 6)):
        gpu.integrate_depth(T, depth, label, cam.K)
        if k in (2, 5):
            gpu.update_mesh()
    v = gpu.mesh_view_device()
    torch.cuda.synchronize()
    v = {k: t.cpu().numpy() for k, t in v.items()}
    layer = gpu.export_mesh()
    nb = len(v["block_keys"])
    assert nb == gpu.num_blocks() == len(layer["block_index"]) and v["block_first"][-1] == len(layer["vertices"])
    bias = 1 << 20
    k = v["block_keys"].astype(np.uint64)
    blocks = np.stack([(k & 0x1FFFFF), (k >> 21) & 0x1FFFFF, (k >> 42) & 0x1FFFFF], 1).astype(np.int64) - bias
    order = np.argsort(v["block_keys"], kind="stable")                   # numeric key order = (z, y, x)
    f = v["block_first"]
    view = {"vertices": np.concatenate([v["vertices"][f[s]:f[s + 1]] for s in order]),
            "rgba": np.concatenate([v["rgba"][f[s]:f[s + 1]] for s in order]),
            "labels": np.concatenate([v["labels"][f[s]:f[s + 1]] for s in order]),
            "block_index": blocks[order].astype(np.int32),
            "block_first": np.concatenate([[0], np.cumsum([f[s + 1] - f[s] for s in order])]).astype(np.int64)}
    _same(view, layer)
    gpu.close()


def test_rejected_inputs():
    cfg = make_config(KSG_INTEGRATOR_FAST, VS, C, max_points=W * H, max_updates=16 << 20)
    gpu = Integrator(cfg)
    lib, h = gpu.lib, gpu.handle
    cam, depth, label, T = next(iter(frames(W, H, C, 1)))
    gpu.integrate_depth(T, depth, label, cam.K)
    n, m = Ct.c_int64(), Ct.c_int64()
    assert lib.ksg_export_mesh(h, 0, 0, None, None, None, 0, None, None, Ct.byref(n), Ct.byref(m)) == 1   # before any update
    assert lib.ksg_mesh_view_device(h, Ct.byref(n), Ct.byref(m), None, None, None, None, None) == 1
    for mw in (float("nan"), -1.0):
        assert lib.ksg_update_mesh(h, mw, None) == 1, mw
        assert lib.ksg_export_mesh(h, 0, 0, None, None, None, 0, None, None, Ct.byref(n), Ct.byref(m)) == 1  # no layer made
    assert lib.ksg_update_mesh(None, 1e-4, None) == 1
    st = KsgMeshStats()
    assert lib.ksg_update_mesh(h, 1e-4, Ct.byref(st)) == 0 and st.full == 1
    assert lib.ksg_export_mesh(h, 0, 0, None, None, None, 0, None, None, Ct.byref(n), Ct.byref(m)) == 0
    assert n.value == st.vertices > 0 and m.value == gpu.num_blocks()
    nv, nb = n.value, m.value
    vtx = np.zeros((nv, 3), F)
    assert lib.ksg_export_mesh(h, 0, nv - 1, vtx.ctypes.data, None, None, 0, None, None, None, None) == 1         # vertex capacity
    first = np.zeros(nb + 1, np.int64)
    assert lib.ksg_export_mesh(h, 0, nv, None, None, None, nb - 1, None, first.ctypes.data, None, None) == 1      # block capacity
    assert lib.ksg_export_mesh(h, 0, -1, None, None, None, 0, None, None, None, None) == 1
    assert lib.ksg_export_mesh(h, 0, nv, vtx.ctypes.data, None, None, 0, None, None, None, None) == 0
    assert vtx.tobytes() == gpu.extract_mesh()["vertices"].tobytes()
    gpu.close()
    sharded = Integrator(make_config(KSG_INTEGRATOR_FAST, VS, C, max_points=1024, max_updates=1 << 16, shard_count=2, shard_rank=1))
    assert sharded.lib.ksg_update_mesh(sharded.handle, 1e-4, None) == 1
    assert b"shard" in sharded.lib.ksg_last_error(sharded.handle)
    sharded.close()


def test_shim_update_mesh_assembles_its_final_mesh(demo, tmp_path):  # noqa: F811
    """shim_demo --mesh-every 2: SemanticTsdfServer::updateMesh after every second frame, its changed blocks assembled into one host
    mesh, equals the final extractMesh; generateMesh's .ply parses to the same soup"""
    w, h, vs = 320, 240, 0.10
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
    want = gpu.extract_mesh()
    fpath, opath, ppath = tmp_path / "frames.bin", tmp_path / "out.bin", tmp_path / "mesh.ply"
    write_frames(fpath, fr, vs, 16, pal, [C - 1])
    env = dict(os.environ, KSG_MAX_POINTS=str(w * h), KSG_MAX_UPDATES=str(8 << 20))
    r = subprocess.run([demo, "fast", str(fpath), str(opath), "lazy", "--mesh-every", "2", str(ppath)],
                       capture_output=True, text=True, env=env, timeout=600)
    assert r.returncode == 0, r.stderr + r.stdout
    assert "mesh-every: 3 updates, assembled mesh equals extractMesh" in r.stdout, r.stdout
    ply = parse_ply(ppath)
    assert ply["vertices"].tobytes() == want["vertices"].tobytes()
    assert ply["rgba"].tobytes() == want["rgba"].tobytes() and ply["labels"].tobytes() == want["labels"].tobytes()
    gpu.close()
