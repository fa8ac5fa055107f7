"""`fast`'s voxel update (k_fast_group + k_fast_apply, ksg_fast.cuh) on a tile that no synthetic depth frame fills: the camera
sits inside one 8^3 tile and rays from every direction end on a sphere around it, so that tile holds more records than one CTA
sorts in shared memory (kFastKeyCap = 4096: its keys are sorted in global memory), all 512 of its voxels are work items, and
the voxel of the camera receives one record per cast ray (hundreds of 32-record batches in one work item).

The CPU test certifies those three properties on the oracle's map (constant weight 1 and no drop-off in free space, so a voxel's
weight after one frame into an empty map is its record count).  The device must then match the oracle bit for bit over two
frames (the second one updates voxels that already hold state), its update log must list every voxel the frame changed, once,
with the state the map holds, and two spatial shards assembled with their ownership masks must give the same map.

Sharded `fast` frames of the synthetic stream are covered by test_gpu_more.py::test_spatially_sharded_map_equals_unsharded, and
saturated voxels with real colours by `fast_saturate` in test_gpu_apply_edges.py.  The item array cannot overflow: it holds
min(record capacity, tile capacity x 512) items, and a frame has at most one item per record and 512 per tile.
"""
import numpy as np
import pytest

from kimera_semantics_b200.capi import KSG_INTEGRATOR_FAST, Integrator, merge_shard_exports
from oracle.oracle_py import OracleIntegrator
from parity_utils import assert_parity, compare_maps, make_config

C = 21
VS = 0.05
N_POINTS = 8000
KEY_CAP = 4096                          # kFastKeyCap
CAMERA = (0.2125, 0.2125, 0.2125)       # centre of voxel (4, 4, 4): inside tile 0 of block (0, 0, 0)


def pose(t):
    return np.array([1, 0, 0, 0, t[0], t[1], t[2]], np.float32)


def scene():
    """(cfg, frames): two frames of N_POINTS points on spheres around the camera, the second from a camera 1.5 voxels away."""
    cfg = make_config(KSG_INTEGRATOR_FAST, VS, C, max_points=N_POINTS, use_const_weight=1, max_weight=1e6,
                      max_consecutive_ray_collisions=100000, max_updates=8 << 20)
    rng = np.random.default_rng(23)
    out = []
    for k, (radius, shift) in enumerate(((1.0, 0.0), (1.2, 1.5 * VS))):
        d = rng.normal(size=(N_POINTS, 3))
        d /= np.linalg.norm(d, axis=1, keepdims=True)
        xyz = (radius * d).astype(np.float32)
        xyz[np.abs(xyz) < 1e-3] = 1e-3     # no exactly-zero ray component (fast_solver_scenes.off_axis)
        labels = rng.integers(0, C - 1, N_POINTS).astype(np.uint8)
        out.append((pose(np.array(CAMERA) + shift), xyz, labels))
    return cfg, out


def camera_tile_counts(exp):
    """Record count of each voxel of the camera's tile (local voxels 0..7 of block (0, 0, 0)), from a one-frame map."""
    b = np.nonzero((exp["block_index"] == 0).all(axis=1))[0]
    assert len(b) == 1
    w = exp["tsdf_weight"][b[0]].reshape(16, 16, 16)      # [z][y][x]
    return w[:8, :8, :8]


def test_dense_tile_scene_reaches_the_edges_cpu():
    cfg, frames = scene()
    ora = OracleIntegrator(cfg)
    T, xyz, labels = frames[0]
    ora.integrate_points(T, xyz, labels=labels)
    counts = camera_tile_counts(ora.export())
    assert np.array_equal(counts, np.round(counts)), "weights are not record counts"
    assert (counts > 0).all(), "not every voxel of the camera's tile is touched"
    assert counts.sum() > KEY_CAP, f"the camera's tile holds {counts.sum()} records, not more than {KEY_CAP}"
    assert counts.max() > 32 * 8, f"the longest voxel segment has {counts.max()} records"


@pytest.mark.gpu
def test_dense_tile_matches_oracle_and_logs_every_changed_voxel():
    cfg, frames = scene()
    gpu, ora = Integrator(cfg), OracleIntegrator(cfg)
    gpu.set_update_log(1 << 20)
    before = None
    for T, xyz, labels in frames:
        before = ora.export()
        sg = gpu.integrate_points(T, xyz, labels=labels)
        so = ora.integrate_points(T, xyz, labels=labels)
        assert sg.voxel_updates == so.voxel_updates and sg.blocks_allocated == so.blocks_allocated
        rep = compare_maps(gpu.export(), ora.export())
        assert_parity(rep, rtol=0.0)
        assert rep["tsdf_distance_bit_mismatch"] == 0 and rep["tsdf_weight_bit_mismatch"] == 0 and rep["sem_priors_bit_mismatch"] == 0
    after, exp = ora.export(), gpu.export()
    heads, priors = gpu.fetch_update_log()
    logged = {(tuple(int(x) for x in h["block_index"]), int(h["lin_label"]) & 0xFFFFFF) for h in heads}
    assert len(logged) == len(heads), "a voxel is logged twice"
    # every voxel the frame changed is logged (a voxel whose records were all skipped for weight is logged too: its row changed
    # or not, it was updated), and every entry is the voxel's state in the map
    prev = {tuple(b): k for k, b in enumerate(before["block_index"])}
    for k, b in enumerate(after["block_index"]):
        k0 = prev.get(tuple(b))
        w0 = before["tsdf_weight"][k0] if k0 is not None else np.zeros_like(after["tsdf_weight"][k])
        p0 = before["sem_priors"][k0] if k0 is not None else None
        moved = after["tsdf_weight"][k] != w0
        if p0 is not None:
            moved |= (after["sem_priors"][k] != p0).any(axis=-1)
        for lin in np.nonzero(moved)[0]:
            assert (tuple(int(x) for x in b), int(lin)) in logged
    row = {tuple(b): k for k, b in enumerate(exp["block_index"])}
    for h, pr in zip(heads, priors):
        k, lin = row[tuple(int(x) for x in h["block_index"])], int(h["lin_label"]) & 0xFFFFFF
        assert h["tsdf_weight"] == exp["tsdf_weight"][k][lin] and h["tsdf_distance"] == exp["tsdf_distance"][k][lin]
        assert np.array_equal(pr, exp["sem_priors"][k][lin])
    gpu.close()


@pytest.mark.gpu
def test_dense_tile_sharded_equals_oracle():
    cfg, frames = scene()
    ora = OracleIntegrator(cfg)
    shards = []
    for r in range(2):
        c, _ = scene()
        c.shard_rank, c.shard_count = r, 2
        shards.append(Integrator(c))
    for T, xyz, labels in frames:
        ora.integrate_points(T, xyz, labels=labels)
        for s in shards:
            s.integrate_points(T, xyz, labels=labels)
    merged = merge_shard_exports([s.export() for s in shards], 16)
    assert_parity(compare_maps(merged, ora.export()), rtol=0.0)
    for s in shards:
        s.close()
