"""tsdf_batch (csrc/ksg_kernels.cuh), the TSDF recurrence of every warp-level apply kernel, on its own on the device
(ksg_debug_tsdf_batch: one warp, batches of 32 as in k_voxel_apply_long) against the sequential float32 definition, bit for bit in
distance, weight and colour, for the plain and the WIDE instance.  The record chains are the families of tests/apply_branch_model.py;
tests/test_apply_branch_model_cpu.py proves which of the kernel's five weight paths and two distance paths each of them takes."""
import numpy as np
import pytest

import apply_branch_model as M
from kimera_semantics_b200.capi import KSG_INTEGRATOR_MERGED, debug_tsdf_batch, default_config

pytestmark = pytest.mark.gpu

FAMILIES = M.families()


def device_result(f, wide):
    cfg = default_config(KSG_INTEGRATOR_MERGED, 0.1, 16, 21)
    cfg.default_truncation_distance = float(f["trunc"])
    cfg.max_weight = float(f["max_weight"])
    return debug_tsdf_batch(cfg, f["sdf"], f["uw"], f["dist"], f["wgt"], rgba=f["rgba"], colors=f["colors"], keep_blend=f["blend"],
                            wide=wide)


@pytest.mark.parametrize("wide", [False, True])
def test_every_family_equals_the_sequential_definition_bit_for_bit(wide):
    bad = []
    for f in FAMILIES:
        got, ref = device_result(f, wide), M.run_sequential(f)
        if not M.same_state(got, ref):
            bad.append((f["name"], [float(got[0]), float(got[1]), hex(int(got[2]))], [float(ref[0]), float(ref[1]), hex(int(ref[2]))]))
    assert not bad, bad


def test_empty_chain_leaves_the_state():
    f = dict(FAMILIES[0], sdf=np.zeros(0, M.F), uw=np.zeros(0, M.F))
    assert M.same_state(device_result(f, False), (f["dist"], f["wgt"], f["rgba"]))
