"""The phases of the `fast` observed-set solver (k_fast_solve3, ksg_fast3.cuh) around the sweeps, at cast-ray counts far from
bench.py's frames, compared with the oracle bit for bit:

- dense: so many isolated points that almost every one is cast, more than one ray per thread of the default solver grid's
  first 32-ray batch per warp (132 CTAs of 32 warps on an H100), so the compaction and the ray set-up loop more than once;
- sparse: a few cast rays spread over a large point capacity, so most 32-point chunks are empty;
- sparse then dense frames into the same map, so the persistent tables and the block probe kept for the key scatter take part.
Every ray of these frames is shorter than the kH0 = 16 steps set up before the first sweep."""
import numpy as np
import pytest

from fast_solver_scenes import off_axis, pose
from gpu_fast_solver_check import parity_failures
from kimera_semantics_b200.capi import KSG_INTEGRATOR_FAST, Integrator
from oracle.oracle_py import OracleIntegrator
from parity_utils import make_config

pytestmark = pytest.mark.gpu

VOXEL = 0.05
LABELS = 5
DENSE = 160_000              # > 32 * 132 * 32 = 135 168 cast rays


def box_points(n, seed, half=(12.0, 12.0, 3.0), near=0.6):
    """n points uniform in a box around the camera, none nearer than `near` (distinct start cells almost surely)."""
    rng = np.random.default_rng(seed)
    p = rng.uniform(-1.0, 1.0, (n, 3)) * np.array(half)
    r = np.linalg.norm(p, axis=1)
    p[r < near] *= (near / np.maximum(r[r < near], 1e-3))[:, None]
    return off_axis(p).astype(np.float32)


def frame(n, seed):
    rng = np.random.default_rng(seed + 100)
    return pose(0.013, -0.021, 0.007), box_points(n, seed), rng.integers(0, LABELS - 1, n).astype(np.uint32), False


def run(frames, max_points):
    cfg = make_config(KSG_INTEGRATOR_FAST, VOXEL, LABELS, max_points=max_points)
    gpu, ora = Integrator(cfg), OracleIntegrator(cfg)
    bad = []
    try:
        for i, fr in enumerate(frames):
            bad += parity_failures(gpu, ora, fr, f"frame {i}")
    finally:
        gpu.close()
    return bad


def test_dense_frame_sets_up_several_batches_per_warp():
    bad = run([frame(DENSE, 1)], DENSE)
    assert not bad, bad


def test_sparse_frame_in_a_large_capacity():
    bad = run([frame(300, 2)], 640 * 480)
    assert not bad, bad


def test_sparse_then_dense_frames_into_one_map():
    bad = run([frame(2000, 3), frame(DENSE, 4), frame(DENSE // 2, 5)], DENSE)
    assert not bad, bad
