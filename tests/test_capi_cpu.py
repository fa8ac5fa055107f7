"""CPU-side checks of the drop-in boundary: the C-ABI library loads, exports every symbol include/ksg.h declares, agrees
with the Python mirror of its structs, rejects bad configs the way the reference CHECKs do, and fails loudly (never
falls back to a CPU path) when there is no CUDA device.  No compute calls are made without a GPU."""
import ctypes as C
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

from kimera_semantics_b200 import capi
from kimera_semantics_b200.capi import (KSG_INTEGRATOR_FAST, KSG_INTEGRATOR_MERGED, KsgConfig, KsgFrameStats, default_config,
                                        load_library)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "ksg.h")


@pytest.fixture(scope="module")
def lib():
    if not os.path.exists(capi.library_path()):
        subprocess.check_call(["make", "-C", os.path.dirname(capi.library_path()), "libksg.so"])
    return load_library()


def declared_functions():
    text = open(HEADER).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(ksg_[a-z_0-9]+)\s*\(", text)))


def test_library_exports_every_declared_symbol(lib):
    names = declared_functions()
    assert len(names) >= 15
    for n in names:
        assert hasattr(lib, n), f"{n} declared in include/ksg.h but not exported by libksg.so"
    assert set(names) == set(capi.KSG_SYMBOLS), set(names) ^ set(capi.KSG_SYMBOLS)
    assert b"sm_90a" in lib.ksg_build_info()


def test_library_contains_sm90a_code_and_tma_instructions():
    out = subprocess.run(["cuobjdump", "-lelf", capi.library_path()], capture_output=True, text=True).stdout
    assert "sm_90a" in out, out
    sass = subprocess.run(["cuobjdump", "-sass", capi.library_path()], capture_output=True, text=True).stdout
    assert "UBLKCP" in sass  # cp.async.bulk (TMA 1-D bulk copy) in the tile kernel


def test_struct_layout_matches_the_c_header(tmp_path):
    src = tmp_path / "sz.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "ksg.h"\nint main(){printf("%zu %zu %zu %zu %zu\\n", sizeof(ksg_config), '
                   'sizeof(ksg_frame_stats), offsetof(ksg_config, label_color), offsetof(ksg_config, device), offsetof(ksg_config, max_ray_steps));return 0;}\n')
    exe = tmp_path / "sz"
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    got = [int(x) for x in subprocess.check_output([str(exe)]).split()]
    want = [C.sizeof(KsgConfig), C.sizeof(KsgFrameStats), KsgConfig.label_color.offset, KsgConfig.device.offset, KsgConfig.max_ray_steps.offset]
    assert got == want


def test_default_config_matches_python_mirror(lib):
    for itype, vs, vps, nl in [(KSG_INTEGRATOR_FAST, 0.05, 16, 21), (KSG_INTEGRATOR_MERGED, 0.02, 32, 150)]:
        c = KsgConfig()
        lib.ksg_default_config(C.byref(c), itype, vs, vps, nl)
        p = default_config(itype, vs, vps, nl)
        skip = {"label_color", "label_color_known", "dynamic_label", "reserved"}
        for name, _ in KsgConfig._fields_:
            if name in skip:
                continue
            assert getattr(c, name) == getattr(p, name), name
        assert c.default_truncation_distance == np.float32(4.0) * np.float32(vs)


@pytest.mark.parametrize("mutate,msg", [
    (lambda c: setattr(c, "abi_version", 99), "abi_version"),
    (lambda c: setattr(c, "integrator_type", 7), "integrator type"),
    (lambda c: setattr(c, "voxels_per_side", 12), "power of two"),
    (lambda c: setattr(c, "num_labels", 1), "num_labels"),
    (lambda c: setattr(c, "semantic_measurement_probability", 0.5), "probability"),   # CHECK_GT(log_match, log_non_match)
    (lambda c: setattr(c, "semantic_measurement_probability", 1.0), "probability"),   # CHECK_LT(match, 1.0)
    (lambda c: setattr(c, "color_mode", 3), "color mode"),
    (lambda c: setattr(c, "max_points", 0), "max_points"),
    (lambda c: setattr(c, "merged_bundle_order", 2), "merged_bundle_order"),
    (lambda c: setattr(c, "hot_voxel_mode", 5), "hot_voxel_mode"),
])
def test_create_rejects_invalid_configs_before_touching_the_device(lib, mutate, msg):
    cfg = default_config()
    mutate(cfg)
    h = C.c_void_p()
    rc = lib.ksg_create(C.byref(cfg), C.byref(h))
    assert rc == 1 and not h.value
    assert msg.lower() in lib.ksg_last_error(None).decode().lower()


@pytest.mark.skipif(torch.cuda.is_available(), reason="only meaningful on a box without a GPU")
def test_no_cpu_fallback_without_a_device(lib):
    h = C.c_void_p()
    rc = lib.ksg_create(C.byref(default_config()), C.byref(h))
    assert rc == 6 and not h.value                      # KSG_ERR_NO_DEVICE
    assert "no cpu fallback" in lib.ksg_last_error(None).decode().lower()
    with pytest.raises(capi.KsgError):
        capi.Integrator(default_config())


def test_null_handles_are_rejected(lib):
    assert lib.ksg_sync(None) == 1
    assert lib.ksg_num_blocks(None) == 0
    assert lib.ksg_reset(None) == 1
    assert lib.ksg_integrate_points(None, None, None, None, None, 0, 0, None) == 1


def test_missing_library_is_an_error_not_a_fallback(tmp_path):
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        load_library(str(tmp_path / "libksg_missing.so"))


def test_owner_masks_partition_every_block(lib):
    """Spatial sharding (SURVEY.md 8e): the per-rank ownership masks are disjoint, cover every voxel, are constant per 8^3 tile
    and depend only on (block index, tile) - every rank computes the same partition without communication."""
    from kimera_semantics_b200.capi import owner_mask
    rng = np.random.default_rng(3)
    bi = rng.integers(-50, 50, size=(40, 3)).astype(np.int32)
    for vps in (4, 8, 16, 32):
        for G in (1, 2, 3, 8):
            masks = [owner_mask(bi, vps, r, G, lib) for r in range(G)]
            total = np.sum(masks, axis=0)
            assert (total == 1).all()
            T = min(vps, 8)
            m0 = masks[0].reshape(len(bi), vps, vps, vps)      # [b, z, y, x]
            tiles = m0.reshape(len(bi), vps // T, T, vps // T, T, vps // T, T)
            assert (tiles.min(axis=(2, 4, 6)) == tiles.max(axis=(2, 4, 6))).all()
            if G > 1 and vps >= 16:
                share = np.array([m.mean() for m in masks])
                assert share.min() > 0.5 / G               # no rank is starved
    assert lib.ksg_owner_mask(12, 0, 2, 0, None, None) == 1   # vps must be a power of two
    cfg = default_config()
    cfg.shard_count, cfg.shard_rank = 2, 2
    h = C.c_void_p()
    assert lib.ksg_create(C.byref(cfg), C.byref(h)) == 1 and b"shard_rank" in lib.ksg_last_error(None)
