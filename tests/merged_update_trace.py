"""The voxels a `merged` frame updates, defined without the CUDA path: the reference for the update log of the merged integrator.

A diff of the map before and after a frame cannot serve: it misses the voxels whose update changed nothing (a saturated voxel at
+truncation, label 0, whose likelihood column is zero).  Which voxels a merged frame updates depends on the frame alone - the bundles,
their rays and the anti-grazing set - never on the map (merged.cpp:97-329).  So the frame is integrated a second time into a FRESH
oracle with every label replaced by 1: every update then adds L[:, 1] * n (n >= 1 points of weight >= kEpsilon in the bundle) to the
voxel's log-probability row, whose entries are all non-zero, so the updated voxels are exactly those whose row is no longer the
constructor's value (semantic_voxel.h:21-23).  tests/test_merged_update_trace_cpu.py checks this definition against a numpy RayCaster
and against the oracle's counters and updated() blocks."""
import numpy as np

from oracle.oracle_py import OracleIntegrator

P_INIT = np.float32(-0.60205999132)     # SemanticVoxel::semantic_priors at construction


def updated_in_export(exp):
    """(block_index [n, 3] int32, linear index [n] int64) of the voxels of a fresh map whose log-probability row has moved."""
    moved = (exp["sem_priors"].view(np.uint32) != P_INIT.view(np.uint32)).any(axis=2)
    b, lin = np.nonzero(moved)
    return exp["block_index"][b], lin.astype(np.int64)


def updated_voxels_points(cfg, T, xyz, labels=None, freespace=False):
    """The voxels `merged` integrate_points(T, xyz, freespace) updates, as (block_index, linear index)."""
    o = OracleIntegrator(cfg)
    try:
        o.integrate_points(T, xyz, labels=np.ones(len(xyz), np.uint8), freespace=freespace)
        return updated_in_export(o.export())
    finally:
        o.close()


def updated_voxels_depth(cfg, T, depth, K):
    """The voxels `merged` integrate_depth(T, depth, label, K) updates, as (block_index, linear index)."""
    o = OracleIntegrator(cfg)
    try:
        o.integrate_depth(T, depth, np.ones(depth.shape, np.uint8), K)
        return updated_in_export(o.export())
    finally:
        o.close()


def pairs(block_index, lin):
    """A set of (bx, by, bz, linear index) tuples."""
    bi = np.asarray(block_index, np.int64).reshape(-1, 3)
    return set(zip(bi[:, 0].tolist(), bi[:, 1].tolist(), bi[:, 2].tolist(), np.asarray(lin, np.int64).tolist()))


def voxel_pairs(vox, vps):
    """Global voxel indices [n, 3] -> set of (block, linear index) tuples (voxblox order: x fastest)."""
    vox = np.asarray(vox, np.int64)
    b = np.floor_divide(vox, vps)
    loc = vox - b * vps
    return pairs(b, loc[:, 0] + vps * (loc[:, 1] + vps * loc[:, 2]))
