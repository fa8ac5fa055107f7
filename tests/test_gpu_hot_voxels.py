"""Opt-in hot-voxel pre-pass of `merged` (ksg_config.hot_voxel_mode = 1, csrc/ksg_hot.cuh): the voxels next to the camera receive
tens of thousands of semantic updates per frame; their per-class float32 addition chains are evaluated as exact scans over
1024-record chunks by many warps instead of one warp's sequential loop.  The map must stay bit-identical to the oracle and the
pre-pass must actually engage.

Status: algorithm proven on the CPU (tools/exact_float_chain.py, csrc/test/chain_host_test.cpp); the GPU check runs in its own
process.  The default path is provably untouched: the SASS
of every existing k_tile_apply instantiation is identical up to one parameter offset.

The frames here never saturate a voxel (max_weight 10000), so mode 2 is checked for parity only; that its skip of a hot voxel at
(+truncation, max_weight) is actually taken, and refused while the distance still moves, is asserted in test_gpu_apply_edges.py."""
import json
import os
import subprocess
import sys

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.mark.gpu
def test_hot_voxel_prepass_keeps_the_map_bit_identical():
    r = subprocess.run([sys.executable, os.path.join(HERE, "gpu_hot_voxel_check.py")], capture_output=True, text=True, timeout=420)
    assert r.returncode == 0, r.stderr[-2000:]
    report = json.loads([l for l in r.stdout.splitlines() if l.startswith("REPORT ")][-1][len("REPORT "):])
    assert len(report) == 4          # canonical / libstdc++ bundle order x mode 1 (semantic rows) / mode 2 (+ TSDF fixed-point check)
    for name, e in report.items():
        assert e["same_blocks"] == 1.0 and e["stats_ok"], (name, e)
        assert not any(v for k, v in e.items() if k.endswith("mismatch")), (name, e)
        assert e["hot_voxels"] > 0, (name, e)
