"""Host paths of an integrator handle that the numeric tests do not reach: a ksg_create that fails after it has allocated, the
pipelined host entry (ksg_integrate_depth_async / ksg_wait_frame), every buffer that grows during a handle's life grown at least
twice, and create / integrate / destroy for every allocation variant.  Results are compared with fresh handles, bit for bit."""
import ctypes as C

import numpy as np
import pytest

from kimera_semantics_b200 import synth
from kimera_semantics_b200.capi import (Integrator, KsgError, KSG_BUNDLE_ORDER_CANONICAL, KSG_BUNDLE_ORDER_LIBSTDCXX,
                                        KSG_INTEGRATOR_FAST, KSG_INTEGRATOR_MERGED, KSG_ORDER_SORTED, _ptr)
from parity_utils import make_config

pytestmark = pytest.mark.gpu
TYPES = [(KSG_INTEGRATOR_FAST, "fast"), (KSG_INTEGRATOR_MERGED, "merged")]


def frame(W, H, C, f):
    cam = synth.make_camera(W, H)
    depth, label, T = synth.frame(cam, f, C)
    return cam, depth, label, T


def stats(st):
    """Frame statistics that two handles fed the same frames must agree on.  Left out: `fast` counts in ray_steps the candidate
    steps its observed-set solver evaluated, and in fixpoint_iterations its sweeps; both depend on the order in which warps claim
    rays (the fixpoint, and so the map, does not)."""
    d = st.as_dict()
    for k in ("ray_steps", "fixpoint_iterations"):
        d.pop(k)
    return d


def integrate(gpu, W, H, C, fs):
    return [stats(gpu.integrate_depth(T, depth, label, cam.K)) for cam, depth, label, T in (frame(W, H, C, f) for f in fs)]


def log_entries(log):
    """(entries, rows) of an update log in (block index, voxel) order: `fast` writes its entries in the order its tile CTAs finish."""
    heads, pri = log
    bi = heads["block_index"]
    order = np.lexsort((heads["lin_label"] & 0xFFFFFF, bi[:, 2], bi[:, 1], bi[:, 0]))
    return heads[order].tobytes(), pri[order].tobytes()


def assert_same_map(a, b, where=""):
    assert a.keys() == b.keys()
    for k in a:
        assert a[k].shape == b[k].shape and np.array_equal(a[k].view(np.uint8), b[k].view(np.uint8)), (where, k)


def export_by_index(gpu, block_index):
    """ksg_export_blocks_by_index: (found, arrays) for the given blocks, absent ones left zero."""
    bi = np.ascontiguousarray(block_index, np.int32)
    n, V, Cn = len(bi), gpu.cfg.voxels_per_side ** 3, gpu.cfg.num_labels
    out = {"tsdf_distance": np.zeros((n, V), np.float32), "tsdf_weight": np.zeros((n, V), np.float32),
           "tsdf_rgba": np.zeros((n, V, 4), np.uint8), "sem_label": np.zeros((n, V), np.uint8),
           "sem_priors": np.zeros((n, V, Cn), np.float32), "sem_rgba": np.zeros((n, V, 4), np.uint8)}
    found = np.zeros(n, np.uint8)
    gpu._check(gpu.lib.ksg_export_blocks_by_index(
        gpu.handle, n, _ptr(bi, C.c_int32), _ptr(found, C.c_uint8), _ptr(out["tsdf_distance"], C.c_float),
        _ptr(out["tsdf_weight"], C.c_float), _ptr(out["tsdf_rgba"], C.c_uint8), _ptr(out["sem_label"], C.c_uint8),
        _ptr(out["sem_priors"], C.c_float), _ptr(out["sem_rgba"], C.c_uint8)), "ksg_export_blocks_by_index")
    return found, out


def test_create_failing_after_allocation_leaves_the_process_usable():
    """ht_cap * 512 tiles >= 2^32: the config passes validation, and ksg_create fails only once its stream and look-up tables exist."""
    cfg = make_config(KSG_INTEGRATOR_FAST, 0.2, 21, vps=64, max_points=320 * 240, max_blocks=(1 << 22) + 1)
    with pytest.raises(KsgError, match="INVALID_ARGUMENT.*max_blocks too large"):
        Integrator(cfg)
    cfg = make_config(KSG_INTEGRATOR_FAST, 0.05, 21, max_points=320 * 240)
    a, b = Integrator(cfg), Integrator(cfg)
    assert integrate(a, 320, 240, 21, range(3)) == integrate(b, 320, 240, 21, range(3))
    assert_same_map(a.export(), b.export())


@pytest.mark.parametrize("itype,name", TYPES)
def test_async_entry_equals_the_synchronous_entry(itype, name):
    """Frame sizes alternate so that both staging slots of the pipelined entry are replaced by larger ones."""
    C_ = 21
    sizes = [(320, 240), (320, 240), (640, 480), (640, 480), (320, 240), (640, 480), (320, 240), (640, 480)]
    cfg = make_config(itype, 0.05, C_, max_points=640 * 480)
    pipe, ref = Integrator(cfg), Integrator(cfg)
    got, want = [], []
    for f, (W, H) in enumerate(sizes):
        cam, depth, label, T = frame(W, H, C_, f)
        pipe.integrate_depth_async(T, depth, label, cam.K)
        if f > 0:
            got.append(stats(pipe.wait_frame()))
        want.append(stats(ref.integrate_depth(T, depth, label, cam.K)))
    got.append(stats(pipe.wait_frame()))
    assert got == want, name
    assert_same_map(pipe.export(), ref.export(), name)


@pytest.mark.parametrize("itype,name", TYPES)
def test_update_log_switched_grown_off_and_on_again(itype, name):
    C_ = 21
    cfg = make_config(itype, 0.05, C_, max_points=320 * 240)
    a, ref = Integrator(cfg), Integrator(cfg)
    ref.set_update_log(1 << 20)
    caps = [1 << 19, 1 << 20, 0, 3 << 19]
    for f, cap in enumerate(caps):
        a.set_update_log(cap)
        cam, depth, label, T = frame(320, 240, C_, f)
        assert stats(a.integrate_depth(T, depth, label, cam.K)) == stats(ref.integrate_depth(T, depth, label, cam.K))
        want = ref.fetch_update_log()
        if cap == 0:
            with pytest.raises(KsgError, match="update log is off"):
                a.fetch_update_log()
            continue
        got = a.fetch_update_log()
        assert len(want[0]) > 1000, name
        assert log_entries(got) == log_entries(want), (name, f)
    assert_same_map(a.export(), ref.export(), name)


@pytest.mark.parametrize("itype,name", TYPES)
def test_export_staging_grows_and_by_index_lookups(itype, name):
    """Exports after 1 and after 10 frames (the staging grows with the map), then by-index exports, dense and with a sparse hit list."""
    C_ = 21
    cfg = make_config(itype, 0.05, C_, max_points=320 * 240)
    a, ref = Integrator(cfg), Integrator(cfg)
    integrate(a, 320, 240, C_, range(1))
    first = a.export()
    integrate(a, 320, 240, C_, range(1, 10))
    integrate(ref, 320, 240, C_, range(10))
    exp, want = a.export(), ref.export()
    assert len(exp["block_index"]) > len(first["block_index"]) > 0, name
    assert_same_map(exp, want, name)
    keys = ["tsdf_distance", "tsdf_weight", "tsdf_rgba", "sem_label", "sem_priors", "sem_rgba"]
    found, dense = export_by_index(a, want["block_index"])
    assert found.all()
    assert_same_map(dense, {k: want[k] for k in keys}, name)
    # every other block, each followed by an absent one (far away), and a last one outside the key range
    idx = want["block_index"][::2]
    rows = []
    for i, b in enumerate(idx):
        rows += [b, [4000, 4000, 4000 + i]]
    query = np.array(rows + [[1 << 22, 0, 0]], np.int32)
    found, sparse = export_by_index(ref, query)
    assert np.array_equal(found, np.array([1, 0] * len(idx) + [0], np.uint8)), name
    for k in keys:
        assert np.array_equal(sparse[k][found == 1].view(np.uint8), want[k][::2].view(np.uint8)), (name, k)
        assert not sparse[k][found == 0].any(), (name, k)


def test_merge_voxels_device_grows_with_the_delta_count():
    """One delta, then three in one call (more entries than before): the same map as merging the four deltas one call at a time."""
    import torch
    W, H, C_ = 320, 240, 21
    cfg = make_config(KSG_INTEGRATOR_FAST, 0.05, C_, max_points=W * H, max_updates=16 << 20)
    src = Integrator(cfg)
    src.set_update_log(1 << 20)
    deltas = []
    for f in range(4):
        src.clear_map()
        integrate(src, W, H, C_, [f])
        n = src.update_log_size()
        upd = torch.zeros(n * 32, dtype=torch.uint8, device="cuda")
        pri = torch.zeros(n * C_, dtype=torch.float32, device="cuda")
        assert src.copy_update_log_device(upd.data_ptr(), pri.data_ptr(), n) == n
        deltas.append((n, upd, pri))
    torch.cuda.synchronize()
    stride = max(n for n, _, _ in deltas)
    upd3 = torch.zeros(3 * stride * 32, dtype=torch.uint8, device="cuda")
    pri3 = torch.zeros(3 * stride * C_, dtype=torch.float32, device="cuda")
    for g, (n, u, p) in enumerate(deltas[1:]):
        upd3[g * stride * 32:g * stride * 32 + n * 32] = u
        pri3[g * stride * C_:g * stride * C_ + n * C_] = p
    torch.cuda.synchronize()
    grown, ref = Integrator(cfg), Integrator(cfg)
    grown.merge_voxels_device([deltas[0][0]], deltas[0][0], deltas[0][1].data_ptr(), deltas[0][2].data_ptr())
    grown.merge_voxels_device([n for n, _, _ in deltas[1:]], stride, upd3.data_ptr(), pri3.data_ptr())
    for n, u, p in deltas:
        ref.merge_voxels_device([n], n, u.data_ptr(), p.data_ptr())
    a, b = grown.export(), ref.export()
    assert len(a["block_index"]) > 0
    assert_same_map(a, b)


VARIANTS = [
    ("fast-mixed", KSG_INTEGRATOR_FAST, 21, {}, {}),
    ("fast-sorted", KSG_INTEGRATOR_FAST, 21, {"integration_order_mode": KSG_ORDER_SORTED}, {}),
    ("fast-C33", KSG_INTEGRATOR_FAST, 33, {}, {}),
    ("fast-profiling", KSG_INTEGRATOR_FAST, 21, {}, {"profiling": True}),
    ("fast-log", KSG_INTEGRATOR_FAST, 21, {}, {"log": True}),
    ("merged-canonical", KSG_INTEGRATOR_MERGED, 21, {"merged_bundle_order": KSG_BUNDLE_ORDER_CANONICAL}, {}),
    ("merged-libstdcxx", KSG_INTEGRATOR_MERGED, 21, {"merged_bundle_order": KSG_BUNDLE_ORDER_LIBSTDCXX}, {}),
    ("merged-sorted", KSG_INTEGRATOR_MERGED, 21, {"integration_order_mode": KSG_ORDER_SORTED}, {}),
    ("merged-hot0", KSG_INTEGRATOR_MERGED, 21, {"hot_voxel_mode": 0}, {}),
    ("merged-hot1", KSG_INTEGRATOR_MERGED, 21, {"hot_voxel_mode": 1}, {}),
    ("merged-hot2", KSG_INTEGRATOR_MERGED, 21, {"hot_voxel_mode": 2}, {}),
    ("merged-apply1", KSG_INTEGRATOR_MERGED, 21, {"apply_mode": 1}, {}),
    ("merged-C33", KSG_INTEGRATOR_MERGED, 33, {}, {}),
    ("merged-profiling", KSG_INTEGRATOR_MERGED, 21, {}, {"profiling": True}),
    ("merged-log", KSG_INTEGRATOR_MERGED, 21, {}, {"log": True}),
]


@pytest.mark.parametrize("name,itype,C_,fields,extra", VARIANTS, ids=[v[0] for v in VARIANTS])
def test_create_integrate_destroy(name, itype, C_, fields, extra):
    """Each allocation variant twice in one process: create, integrate one frame, export, destroy; both runs agree."""
    cfg = make_config(itype, 0.05, C_, max_points=320 * 240, **fields)
    runs = []
    for _ in range(2):
        gpu = Integrator(cfg)
        if extra.get("profiling"):
            gpu.set_profiling(True)
        if extra.get("log"):
            gpu.set_update_log(1 << 20)
        st = integrate(gpu, 320, 240, C_, [0])[0]
        assert st["voxel_updates"] > 0 and gpu.num_blocks() > 0, name
        if extra.get("profiling"):
            assert gpu.get_profile()["frames"] == 1, name
        if extra.get("log"):
            assert len(gpu.fetch_update_log()[0]) > 0, name
        runs.append((st, gpu.export()))
        gpu.close()
    assert runs[0][0] == runs[1][0], name
    assert_same_map(runs[0][1], runs[1][1], name)
