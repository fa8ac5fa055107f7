"""ksg_integrate_image: the depth / semantic encodings of the reference's front end (kimera_semantics_ros/include/kimera_semantics_ros/
depth_map_to_pointcloud.h:183-193,213-266): float32 metre or uint16 millimetre depth (DepthTraits<T>) and a label image or an RGB semantic
image whose colours name the labels.  The oracle gets the cloud the reference's PointCloudFromDepth::convert<T> would hand to
integratePointCloud (numpy float32 in the reference's operation order) through its points entry; the CUDA path gets the raw images.
The points entry's colour -> label lookup is checked with a table of the largest size, whose lookups walk probe chains."""
import numpy as np
import pytest

from kimera_semantics_b200 import synth
from kimera_semantics_b200.capi import (Integrator, KSG_INTEGRATOR_FAST, KSG_INTEGRATOR_MERGED, KSG_COLOR_MODE_COLOR,
                                        KSG_COLOR_MODE_SEMANTIC, KSG_ORDER_SORTED)
from oracle.oracle_py import OracleIntegrator
from parity_utils import assert_parity, compare_maps, make_config, stats_equal

pytestmark = pytest.mark.gpu

MAX_COLORS = 512   # the largest colour table ksg_set_color_to_label takes


def reference_cloud(depth: np.ndarray, K64):
    """PointCloudFromDepth::convert<T> (depth_map_to_pointcloud.h:222-266) for T = float (metres) or uint16_t (millimetres), and the
    finite filter of the cloud conversion."""
    h, w = depth.shape
    mm = depth.dtype == np.uint16
    fx, fy, cx, cy = [float(x) for x in K64]
    center_x, center_y = np.float32(cx), np.float32(cy)
    unit = float(np.float32(0.001)) if mm else 1.0       # double unit_scaling = DepthTraits<T>::toMeters(1)
    constant_x, constant_y = np.float32(unit / fx), np.float32(unit / fy)
    v, u = np.mgrid[0:h, 0:w]
    d = depth.astype(np.float32)
    x = ((u.astype(np.float32) - center_x) * d).astype(np.float32) * constant_x
    y = ((v.astype(np.float32) - center_y) * d).astype(np.float32) * constant_y
    z = d * np.float32(0.001) if mm else d
    ok = (depth.reshape(-1) != 0) if mm else np.isfinite(depth.reshape(-1))
    xyz = np.stack([x.reshape(-1), y.reshape(-1), z.reshape(-1)], axis=1).astype(np.float32)
    return np.ascontiguousarray(xyz[ok]), np.nonzero(ok)[0]


def color_table(pal: np.ndarray, C: int, size: int):
    """The palette's first C colours with their labels, then (size > C) distinct other colours with labels drawn in [0, C)."""
    rgb, lab = pal[:C, :3].copy(), np.arange(C, dtype=np.uint8)
    if size > C:
        rng = np.random.default_rng(size)
        seen = {tuple(c) for c in rgb} | {(1, 2, 3)}
        extra = []
        while len(extra) < size - C:
            c = tuple(int(x) for x in rng.integers(0, 256, 3))
            if c not in seen:
                seen.add(c)
                extra.append(c)
        rgb = np.concatenate([rgb, np.array(extra, np.uint8)])
        lab = np.concatenate([lab, rng.integers(0, C, size - C).astype(np.uint8)])
    return rgb, lab


def displaced_keys(rgb: np.ndarray) -> int:
    """Keys of the device's 1024-slot open addressing table (home slot (rgb * 2654435761) >> 22, linear probe) that sit behind their
    home slot, i.e. whose lookup walks a probe chain."""
    slots = np.full(1024, -1, np.int64)
    displaced = 0
    for r, g, b in rgb.astype(np.uint32):
        key = int(r | (g << 8) | (b << 16))
        p = ((key * 2654435761) & 0xFFFFFFFF) >> 22
        while slots[p] not in (-1, key):
            p = (p + 1) & 1023
        displaced += int(p != ((key * 2654435761) & 0xFFFFFFFF) >> 22)
        slots[p] = key
    return displaced


# ids 1-1, 1-0, 0-1: (integrator, colour mode) of the uint16 + RGB cases this test started with
CASES = [pytest.param(KSG_INTEGRATOR_FAST, KSG_COLOR_MODE_SEMANTIC, "u16", "rgb", {}, id="1-1"),
         pytest.param(KSG_INTEGRATOR_FAST, KSG_COLOR_MODE_COLOR, "u16", "rgb", {}, id="1-0"),
         pytest.param(KSG_INTEGRATOR_MERGED, KSG_COLOR_MODE_SEMANTIC, "u16", "rgb", {}, id="0-1")]
CASES += [pytest.param(itype, KSG_COLOR_MODE_SEMANTIC, depth, semantic, {}, id=f"{name}-{depth}-{semantic}")
          for itype, name in ((KSG_INTEGRATOR_FAST, "fast"), (KSG_INTEGRATOR_MERGED, "merged"))
          for depth, semantic in (("f32", "label"), ("f32", "rgb"), ("u16", "label"))]
CASES += [pytest.param(itype, KSG_COLOR_MODE_SEMANTIC, "u16", "rgb", {"integration_order_mode": KSG_ORDER_SORTED}, id=f"{name}-sorted")
          for itype, name in ((KSG_INTEGRATOR_FAST, "fast"), (KSG_INTEGRATOR_MERGED, "merged"))]
# merged ignores dynamic labels (only fast.cpp:76 applies isSemanticLabelValid): a third of the labels dynamic on both integrators
CASES += [pytest.param(itype, KSG_COLOR_MODE_SEMANTIC, "f32", "label", {"dynamic": True}, id=f"{name}-dynamic")
          for itype, name in ((KSG_INTEGRATOR_FAST, "fast"), (KSG_INTEGRATOR_MERGED, "merged"))]


@pytest.mark.parametrize("itype,color_mode,depth_type,semantic,kw", CASES)
def test_uint16_depth_and_rgb_semantic_image_entry_matches_the_reference_front_end(itype, color_mode, depth_type, semantic, kw):
    """Every depth x semantic encoding on both integrators (the name is that of the first cases)."""
    W, H, C = 320, 240, 21
    cam = synth.make_camera(W, H)
    kw = dict(kw)
    dynamic = kw.pop("dynamic", False)
    cfg = make_config(itype, 0.05, C, max_points=W * H, max_updates=16 << 20, color_mode=color_mode, **kw)
    if dynamic:
        for l in range(1, C, 3):
            cfg.dynamic_label[l] = 1
    pal = np.array([[cfg.label_color[l][k] for k in range(4)] for l in range(256)], np.uint8)
    table_rgb, table_lab = color_table(pal, C, C)
    gpu, ora = Integrator(cfg), OracleIntegrator(cfg)
    gpu.set_color_to_label(table_rgb, table_lab)
    ora.set_color_to_label(table_rgb, table_lab)
    K64 = np.array([float(cam.K[0]), float(cam.K[1]), float(cam.K[2]), float(cam.K[3])], np.float64)
    for f in range(3):
        depth, label, T = synth.frame(cam, f, C)
        if depth_type == "u16":
            depth = np.clip(np.rint(depth.astype(np.float64) * 1000.0), 0, 65535).astype(np.uint16)
            depth.reshape(-1)[(f * 7)::53] = 0                # invalid measurements
        else:
            depth = depth.copy()
            depth.reshape(-1)[(f * 7)::53] = np.nan
        if semantic == "rgb":
            sem = np.ascontiguousarray(pal[label][:, :, :3])
            sem.reshape(-1, 3)[(f * 5)::97] = (1, 2, 3)       # colours that are not in the table -> label 0 (color.cpp:75-80)
        else:
            sem = label
        sg = gpu.integrate_image(T, depth, sem, K64)
        xyz, pix = reference_cloud(depth, K64)
        if semantic == "rgb":
            rgba = np.concatenate([sem.reshape(-1, 3)[pix], np.full((len(pix), 1), 255, np.uint8)], axis=1)
            so = ora.integrate_points(T, xyz, rgba=np.ascontiguousarray(rgba))
        else:
            so = ora.integrate_points(T, xyz, labels=np.ascontiguousarray(label.reshape(-1)[pix]))
        assert (sg.points_in, sg.points_valid, sg.voxel_updates, sg.rays_cast) == (so.points_in, so.points_valid, so.voxel_updates, so.rays_cast), \
            (sg.as_dict(), so.as_dict())
    assert_parity(compare_maps(gpu.export(), ora.export()))
    gpu.close(); ora.close()


@pytest.mark.parametrize("itype", [KSG_INTEGRATOR_FAST, KSG_INTEGRATOR_MERGED])
def test_points_entry_labels_by_colour_from_a_full_table_match_the_oracle(itype):
    W, H, C = 320, 240, 21
    cam = synth.make_camera(W, H)
    cfg = make_config(itype, 0.05, C, max_points=W * H, max_updates=16 << 20)
    pal = np.array([[cfg.label_color[l][k] for k in range(4)] for l in range(256)], np.uint8)
    table_rgb, table_lab = color_table(pal, C, MAX_COLORS)
    assert displaced_keys(table_rgb) > 100
    gpu, ora = Integrator(cfg), OracleIntegrator(cfg)
    gpu.set_color_to_label(table_rgb, table_lab)
    ora.set_color_to_label(table_rgb, table_lab)
    rng = np.random.default_rng(1)
    for f in range(3):
        depth, label, T = synth.frame(cam, f, C)
        xyz, pix = synth.backproject(depth, cam)
        rgba = pal[label.reshape(-1)[pix]].copy()
        pick = rng.random(len(pix)) < 0.5                     # half of the points carry a colour of anywhere in the table
        rgba[pick, :3] = table_rgb[rng.integers(0, MAX_COLORS, int(pick.sum()))]
        rgba[::97] = (1, 2, 3, 255)                           # not in the table -> label 0
        sg, so = gpu.integrate_points(T, xyz, rgba=rgba), ora.integrate_points(T, xyz, rgba=rgba)
        ok, why = stats_equal(sg, so)
        assert ok, f"frame {f}: {why}"
    assert_parity(compare_maps(gpu.export(), ora.export()))
    gpu.close(); ora.close()
