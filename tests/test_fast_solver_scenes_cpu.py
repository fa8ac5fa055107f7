"""The scenes of tests/fast_solver_scenes.py reach the observed-set solver's rare paths: every certificate is checked against the
threshold of its path, so a builder that stops reaching it fails here, without a GPU.  The oracle and the numpy replay of the `fast`
control flow also agree on every scene (updates, rays cast and touched voxels), so the scenes are what the GPU tests take them for."""
import numpy as np
import pytest

import fast_solver_scenes as S
from kimera_semantics_b200.capi import KSG_INTEGRATOR_FAST
from oracle.oracle_py import OracleIntegrator
from parity_utils import make_config
from test_oracle_crosscheck import FastReplay, touched_voxels


@pytest.fixture(scope="module")
def scenes():
    return {
        "aliased_start": S.scene_aliased_start(),
        "overflow_fan": S.scene_overflow("fan"),
        "overflow_alias": S.scene_overflow("alias"),
        "window_edges_c0": S.scene_window_edges(0),
        "window_edges_c2": S.scene_window_edges(2),
        "deep_fixpoint": S.scene_deep_fixpoint(),
    }


def test_aliased_start_cells_share_a_slot_with_more_visitors_than_one_warp_sorts(scenes):
    cfg, frames, cert = scenes["aliased_start"]
    assert [c["start_slot_visitors"] for c in cert] == list(S.START_VISITORS)
    assert all(c["start_slot_cells"] == 2 for c in cert)
    visitors = [c["start_slot_visitors"] for c in cert]
    assert min(visitors) < S.SORT_PER_WARP < max(visitors)          # both the shared-memory and the in-place sort
    assert S.SORT_PER_WARP in visitors and S.SORT_PER_WARP + 1 in visitors
    assert all(c["rays"] >= 16 for c in cert)                       # a ray at every change of cell in sequence order


@pytest.mark.parametrize("case", ["fan", "alias"])
def test_overflowing_buckets(scenes, case):
    cfg, frames, cert = scenes["overflow_" + case]
    assert len(frames) >= 3
    first = cert[0]
    assert first["max_entries"] >= 1000 and first["slots_over_bucket"] >= 50
    # every candidate of a frame fits the overflow pool, so the longest chain (max_entries - 32) does too
    assert all(c["candidates"] < S.overflow_cap(cfg) for c in cert)
    if case == "alias":
        assert all(c["mixed_slots_over_bucket"] >= 20 for c in cert)     # far voxels with other values in overflowing slots
    assert all(c["table_collisions"] > 0 for c in cert[1:])              # the persistent table decides collisions


@pytest.mark.parametrize("max_collisions", [0, 2])
def test_breaks_at_the_window_edges(scenes, max_collisions):
    cfg, frames, cert = scenes[f"window_edges_c{max_collisions}"]
    assert all(n >= 1 for n in cert[0]["edge_hist"].values()), cert[0]["edge_hist"]
    assert max(cert[0]["lengths"]) > 6 * S.WINDOW
    assert all(c["table_collisions"] > 0 for c in cert[1:])


# the deepest Jacobi iteration a search over planar fans found (S.DEEP); the 64 the code suggests was not reached by a fan
DEEP_SWEEPS = 20


def test_deep_fixpoint_needs_many_jacobi_sweeps(scenes):
    cfg, frames, cert = scenes["deep_fixpoint"]
    assert cert[0]["sweeps"] >= DEEP_SWEEPS
    assert cert[0]["rays"] > 150
    assert all(c["table_collisions"] > 0 for c in cert[1:])


@pytest.mark.parametrize("name", ["aliased_start", "overflow_fan", "overflow_alias", "window_edges_c0", "window_edges_c2", "deep_fixpoint"])
def test_oracle_and_replay_agree(scenes, name):
    cfg, frames, cert = scenes[name]
    assert all(c["zero_ray_components"] == 0 for c in cert)      # the reference leaves such rays unspecified
    ora, rep = OracleIntegrator(cfg), FastReplay(cfg)
    for i, (T, xyz, labels, freespace) in enumerate(frames):
        so = ora.integrate_points(T, xyz, labels=labels, freespace=freespace)
        valid, rays, updates = rep.integrate(T, xyz, labels)
        assert (valid, rays, updates) == (so.points_valid, so.rays_cast, so.voxel_updates), f"frame {i}"
        assert (rays, updates) == (cert[i]["rays"], sum(cert[i]["U"])), f"frame {i}: the certificate models another frame"
    tv = touched_voxels(ora.export(), cfg.voxels_per_side)
    assert tv <= rep.touched and len(rep.touched) - len(tv) <= 0.02 * len(rep.touched) + 5
