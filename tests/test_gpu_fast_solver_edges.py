"""The `fast` observed-set solver (k_fast_solve3, ksg_fast3.cuh) on the scenes of tests/fast_solver_scenes.py, which reach its rare
paths: shared start-set slots with more than 1024 visitors, overflowing buckets, breaks at the 64-step block edges, deep
fixpoints and their worklist sweeps, and the persistent table across frames, resets and cleared maps.

Every frame is compared with the oracle bit for bit under three solver block sizes (KSG_SOLVE_THREADS 1024, 512, 256: warps per
CTA and CTAs per SM change, and with them the interleaving of the sweeps).  Each shape runs once, in its own process, so the
variable does not leak into other tests.  A profiled run then shows on the device that each path was taken.  The error paths
(scratch exhausted, voxel index out of range) must be reported, stay reported until reset(), and leave a clean integrator after it."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

import fast_solver_scenes as S
from kimera_semantics_b200.capi import Integrator, KsgError
from oracle.oracle_py import OracleIntegrator
from gpu_fast_solver_check import parity_failures

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
SCENES = ("aliased_start", "aliased_start_sorted", "overflow_fan", "overflow_alias", "window_edges_c0", "window_edges_c2",
          "deep_fixpoint")


def run_helper(mode, threads=None):
    env = dict(os.environ)
    env.pop("KSG_SOLVE_THREADS", None)
    if threads is not None:
        env["KSG_SOLVE_THREADS"] = str(threads)
    r = subprocess.run([sys.executable, os.path.join(HERE, "gpu_fast_solver_check.py"), mode], capture_output=True, text=True,
                       timeout=600, env=env)
    assert r.returncode == 0, r.stderr[-2000:]
    line = [l for l in r.stdout.splitlines() if l.startswith("REPORT ")][-1]
    report = json.loads(line[len("REPORT "):])
    assert sorted(report) == sorted(SCENES)
    return report


@pytest.mark.parametrize("threads", [1024, 512, 256])
def test_scenes_bit_exact_under_each_solver_shape(threads):
    report = run_helper("parity", threads)
    bad = {k: v for k, v in report.items() if v}
    assert not bad, bad


def test_scenes_reach_their_paths_on_the_device():
    """Frame 0 of each scene.  The later, overlapping frames exercise the persistent table, but the start set keeps most of
    their points from casting (the previous frame's offset aliases the neighbouring cell, A.4): they converge in 2-3 sweeps
    and break at few of the window edges, so the worklist and the edge steps are asserted on frame 0 only."""
    report = run_helper("coverage")
    jacobi = {name: build(certificate=True)[2][0]["sweeps"] for name, build in
              (("window_edges_c0", lambda **k: S.scene_window_edges(0, **k)), ("window_edges_c2", lambda **k: S.scene_window_edges(2, **k)),
               ("deep_fixpoint", S.scene_deep_fixpoint))}
    print("device coverage:", json.dumps(report))
    print("CPU Jacobi sweeps of frame 0:", json.dumps(jacobi))
    for name in ("aliased_start", "aliased_start_sorted"):      # phase 0b sorts in shared memory up to 1024, in place beyond
        assert [f["max_shared_slot_visitors"] for f in report[name]] == list(S.START_VISITORS), report[name]
    for name, cpu_sweeps in jacobi.items():
        first = report[name][0]
        assert 4 <= first["sweeps"] <= first["rays"] + 2, (name, first, cpu_sweeps)   # past sweep 3: the worklist runs
        assert first["rays_scanned"] < first["rays"] * first["sweeps"], (name, first)
    for frames in report.values():
        assert all(f["sweeps"] <= f["rays"] + 2 for f in frames)


def frame_parity(gpu, ora, frame, where):
    bad = parity_failures(gpu, ora, frame, where)
    assert not bad, bad


def test_deepest_fan_converges_under_the_tightest_sweep_budget():
    """The deepest fan with max_points = its point count, the tightest budget (max_points + 2 sweeps) a frame of it can have.
    This checks convergence, parity and the bound on the sweeps the device takes; it cannot make the budget run out, because
    the budget is the proven bound: a frame of R <= max_points rays converges within R + 2 sweeps (DESIGN.md section 4)."""
    cfg, frames, _ = S.scene_deep_fixpoint(certificate=False)
    cfg.max_points = len(frames[0][1])
    gpu, ora = Integrator(cfg), OracleIntegrator(cfg)
    gpu.set_profiling(True)
    for i, frame in enumerate(frames):
        frame_parity(gpu, ora, frame, f"frame {i}")
        tl = gpu.fast_timeline()
        assert 1 <= tl["sweeps"] <= tl["debug"]["rays"] + 2 <= cfg.max_points + 2, tl
    gpu.close()


def expect_sticky(gpu, frame, status):
    """The frame's error is reported by the frame's call or, at the latest, by sync(); every later call reports it again."""
    T, xyz, labels, freespace = frame
    with pytest.raises(KsgError, match=status):
        gpu.integrate_points(T, xyz, labels=labels, freespace=freespace)
        gpu.sync()
    with pytest.raises(KsgError, match=status):
        gpu.integrate_points(T, xyz, labels=labels, freespace=freespace)
    with pytest.raises(KsgError, match=status):
        gpu.sync()


def pairs_only(frame):
    """The ten window-edge rays without the fan: a frame that fits the scratch of the test below."""
    T, xyz, labels, freespace = frame
    n = 2 * len(S.WINDOW_EDGE_STEPS)
    return T, xyz[:n], labels[:n], freespace


def test_scratch_full_is_reported_and_sticky_until_reset():
    cfg, frames, _ = S.scene_window_edges(2, certificate=False)
    cfg.max_ray_steps = 20000          # the fan's ~90 K candidate steps do not fit, the ten pairs' ~5 K do
    gpu = Integrator(cfg)
    expect_sticky(gpu, frames[0], "SCRATCH_FULL")
    gpu.reset()
    ora = OracleIntegrator(cfg)
    for i, frame in enumerate(frames):
        frame_parity(gpu, ora, pairs_only(frame), f"after reset, frame {i}")
    gpu.close()


INSIDE = ((1 << 20) - 120, (1 << 20) - 76)   # voxel index of the camera on x and y: the scene reaches 15-20 voxels from +-2^20


@pytest.mark.parametrize("sign", [(1, -1), (-1, 1)])
def test_scene_just_inside_the_index_range_is_bit_exact(sign):
    """Voxel indices within a few voxels of +-2^20 on x and y, through the worklist sweeps of the window-edge scene: index_hash
    and pack_key on large positive and negative coordinates."""
    origin = (sign[0] * INSIDE[0] * 0.01, sign[1] * INSIDE[1] * 0.01, 0.0)
    cfg, frames, _ = S.scene_window_edges(2, origin=origin, certificate=False)
    gpu, ora = Integrator(cfg), OracleIntegrator(cfg)
    for i, frame in enumerate(frames):
        frame_parity(gpu, ora, frame, f"frame {i}")
    b = ora.export()["block_index"].astype(np.int64)
    vps = cfg.voxels_per_side
    lo, hi = b[:, :2].min(axis=0) * vps, b[:, :2].max(axis=0) * vps + vps - 1     # voxel index range of the allocated blocks
    edge = np.where(np.array(sign) > 0, (1 << 20) - 1 - hi, lo + (1 << 20))
    assert (edge < 32).all(), edge                                               # the map reaches the edge of the range
    gpu.close()


OUTSIDE = [(((1 << 20) + 200) * 0.01, 0.0, 0.0), (0.0, -((1 << 20) + 200) * 0.01, 0.0)]


@pytest.mark.parametrize("origin", OUTSIDE)
def test_scene_outside_the_index_range_is_reported_and_sticky_until_reset(origin):
    cfg, frames, _ = S.scene_window_edges(2, origin=origin, certificate=False)
    gpu = Integrator(cfg)
    expect_sticky(gpu, frames[0], "INDEX_RANGE")
    gpu.reset()
    assert gpu.num_blocks() == 0
    gpu.sync()                         # the status is cleared
    gpu.close()


@pytest.mark.parametrize("origin", OUTSIDE)
def test_reset_after_an_index_range_error_is_a_fresh_integrator(origin):
    cfg, frames, _ = S.scene_window_edges(2, origin=origin, certificate=False)
    gpu = Integrator(cfg)
    expect_sticky(gpu, frames[0], "INDEX_RANGE")
    gpu.reset()
    cfg_in, frames_in, _ = S.scene_window_edges(2, certificate=False)
    ora = OracleIntegrator(cfg_in)
    for i, frame in enumerate(frames_in):
        frame_parity(gpu, ora, frame, f"after reset, frame {i}")
    gpu.close()
