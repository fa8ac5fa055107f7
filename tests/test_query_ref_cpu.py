"""CPU checks of the point-query twin (tests/query_ref.py) against independent references - scipy's trilinear interpolator, analytic
planes and spheres - and of its conventions at ties and for missing / unobserved / invalid input; plus the ctypes mirror of
ksg_query_out against the C header.  The GPU kernel is compared with this twin bit for bit in tests/test_gpu_query.py."""
import ctypes as C
import os
import subprocess

import numpy as np
from scipy.interpolate import RegularGridInterpolator

import mesh_ref as mr
import query_ref as qr
from kimera_semantics_b200.capi import QUERY_FIELDS, KsgQueryOut

F = np.float32
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _grid(exp, vps, lo, hi):
    """dense [z, y, x] distance array of the blocks lo <= index < hi (all present) and the float64 voxel-centre axis"""
    m = (hi - lo) * vps
    D = np.zeros((m, m, m), np.float64)
    for b, d in zip(exp["block_index"], exp["tsdf_distance"]):
        o = (np.asarray(b) - lo) * vps
        D[o[2]:o[2] + vps, o[1]:o[1] + vps, o[0]:o[0] + vps] = d.reshape(vps, vps, vps)
    return D


def test_trilinear_distance_equals_scipy_on_a_random_field():
    vs, vps, lo, hi = 0.1, 4, -1, 2
    rng = np.random.default_rng(1)
    exp = mr.sdf_export(lambda x, y, z: rng.uniform(-0.2, 0.2, x.shape).astype(F), vs, vps, lo, hi)
    D = _grid(exp, vps, lo, hi)
    axis = (np.arange(lo * vps, hi * vps) + 0.5) * vs
    ref = RegularGridInterpolator((axis, axis, axis), D, method="linear")
    p = rng.uniform(axis[0] + 1e-4, axis[-1] - 1e-4, (4000, 3)).astype(F)
    got = qr.query(exp, vs, vps, p)
    assert (got["flags"] & qr.INTERPOLATED).all()
    want = ref(p.astype(np.float64)[:, ::-1])
    assert np.abs(got["distance"] - want).max() <= 1e-5 * vs


def test_plane_distance_and_gradient_are_exact_up_to_rounding():
    vs, vps = 0.1, 8
    n = np.array([0.3, -0.5, 0.81])
    n /= np.linalg.norm(n)
    nf = n.astype(F)
    exp = mr.sdf_export(lambda x, y, z: nf[0] * x + nf[1] * y + nf[2] * z - F(0.05), vs, vps, -1, 2)
    rng = np.random.default_rng(2)
    p = rng.uniform(-vps * vs + 2 * vs, 2 * vps * vs - 2 * vs, (3000, 3)).astype(F)
    got = qr.query(exp, vs, vps, p)
    assert (got["flags"] == 15).all()
    ana = p.astype(np.float64) @ nf.astype(np.float64) - np.float64(F(0.05))
    dmax = np.abs(exp["tsdf_distance"]).max()
    assert np.abs(got["distance"] - ana).max() <= 8 * np.spacing(F(dmax))
    assert np.abs(got["gradient"] - nf).max() < 1e-5


def test_sphere_error_is_of_order_vs_squared_over_r():
    vs, vps, R = 0.05, 8, 0.6
    exp = mr.sdf_export(lambda x, y, z: np.sqrt(x * x + y * y + z * z) - F(R), vs, vps, -3, 3)
    rng = np.random.default_rng(3)
    u = rng.normal(size=(3000, 3))
    u /= np.linalg.norm(u, axis=1, keepdims=True)
    p = (u * rng.uniform(R - 3 * vs, R + 3 * vs, (3000, 1))).astype(F)
    got = qr.query(exp, vs, vps, p)
    assert (got["flags"] == 15).all()
    r = np.linalg.norm(p.astype(np.float64), axis=1)
    assert np.abs(got["distance"] - (r - R)).max() < vs * vs / R
    g = got["gradient"].astype(np.float64)
    assert np.abs(g - p / r[:, None]).max() < 2 * vs / R


def test_ties_on_faces_and_centres():
    vs, vps = 0.1, 8
    exp = mr.sdf_export(lambda x, y, z: x + F(2) * y - z, vs, vps, -3, 2)
    k = np.arange(-22, 14)
    # on a voxel face the point belongs to the upper voxel; at some negative k, fl(fl(k vs) / vs) < k and only the 1e-6 lifts it back
    face = np.stack([F(k) * F(vs) for k in k]).astype(F)
    assert (face * F(1.0 / vs) < k).any()
    yc = F(0.5) * F(vs)                     # centre of voxel 0 in y and z
    p = np.stack([face, np.full_like(face, yc), np.full_like(face, yc)], axis=1)
    got = qr.query(exp, vs, vps, p)
    assert (got["flags"] == 15).all()
    assert np.array_equal(got["tsdf_rgba"][:, 0], (k & (vps - 1)).astype(np.uint8))      # sdf_export: red = linear voxel index
    assert np.array_equal(got["tsdf_distance"], ((k.astype(F) + F(0.5)) * F(vs) + F(2) * yc) - yc)
    # block faces at negative indices: k = -8, -16 start blocks -1, -2 (local index 0)
    bf = np.isin(k, [-16, -8])
    assert bf.sum() == 2
    assert (got["tsdf_rgba"][bf, 0] == 0).all()
    # exactly on a centre: q = 0, the trilinear distance is the voxel's own distance, bit for bit
    g = np.array([[-13, 2, 5], [0, 0, 0], [-17, -9, -20], [7, -1, 3]])
    c = ((g.astype(F) + F(0.5)) * F(vs)).astype(F)
    got = qr.query(exp, vs, vps, c)
    assert (got["flags"] == 15).all()
    assert np.array_equal(got["distance"].view(np.uint32), got["tsdf_distance"].view(np.uint32))


def test_flags_for_missing_unobserved_and_invalid_points():
    vs, vps = 0.1, 4
    exp = mr.sdf_export(lambda x, y, z: y - F(0.01), vs, vps, -1, 1)
    # a point well inside block (0, 0, 0) next to block (-1, 0, 0)
    p0 = np.array([[0.01, 0.2, 0.2]], F)
    assert qr.query(exp, vs, vps, p0)["flags"][0] == 15
    # drop block (-1, 0, 0): the point's voxel stays, its interpolation and gradient lose corners
    keep = ~np.all(exp["block_index"] == (-1, 0, 0), axis=1)
    cut = {k: v[keep] for k, v in exp.items()}
    got = qr.query(cut, vs, vps, p0)
    assert got["flags"][0] == qr.ALLOCATED | qr.OBSERVED
    assert np.isnan(got["distance"][0]) and np.isnan(got["gradient"][0]).all()
    assert got["distance"].view(np.uint32)[0] == qr.NAN_BITS
    # one unobserved corner (weight 0 < min_weight): the voxel holding p0's neighbour (-1, 2, 2) in block (-1, 0, 0)
    unobs = {k: v.copy() for k, v in exp.items()}
    b = int(np.nonzero(np.all(exp["block_index"] == (-1, 0, 0), axis=1))[0][0])
    unobs["tsdf_weight"][b, 3 + vps * (2 + vps * 2)] = 0.0
    got = qr.query(unobs, vs, vps, p0)
    assert got["flags"][0] == qr.ALLOCATED | qr.OBSERVED
    # ... and the point inside that voxel: allocated, not observed, its fields still written
    p1 = np.array([[-0.05, 0.25, 0.25]], F)
    got = qr.query(unobs, vs, vps, p1)
    assert got["flags"][0] == qr.ALLOCATED and got["tsdf_weight"][0] == 0.0 and got["sem_label"][0] == exp["sem_label"][b, 3 + vps * 10]
    # unallocated space, non-finite and out-of-range points: nothing valid, NaN / 0 everywhere
    bad = np.array([[5.0, 5.0, 5.0], [np.nan, 0, 0], [0, np.inf, 0], [0, 0, -np.inf], [1e12, 0, 0], [0, 0, 2e8]], F)
    got = qr.query(exp, vs, vps, bad)
    assert (got["flags"] == 0).all()
    for k in ("tsdf_distance", "tsdf_weight", "distance"):
        assert (got[k].view(np.uint32) == qr.NAN_BITS).all()
    assert (got["gradient"].view(np.uint32) == qr.NAN_BITS).all()
    assert (got["tsdf_rgba"] == 0).all() and (got["sem_label"] == 0).all() and (got["sem_rgba"] == 0).all()


def test_query_out_mirror_matches_the_c_header(tmp_path):
    src = tmp_path / "q.c"
    fields = ", ".join(f"offsetof(ksg_query_out, {f})" for f in QUERY_FIELDS)
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "ksg.h"\nint main(){size_t v[] = {sizeof(ksg_query_out), ' + fields +
                   '}; for (size_t i = 0; i < sizeof(v) / sizeof(v[0]); ++i) printf("%zu ", v[i]); printf("%d %d %d %d\\n", KSG_QUERY_ALLOCATED, '
                   'KSG_QUERY_OBSERVED, KSG_QUERY_INTERPOLATED, KSG_QUERY_GRADIENT); return 0;}\n')
    exe = tmp_path / "q"
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    got = [int(x) for x in subprocess.check_output([str(exe)]).split()]
    want = [C.sizeof(KsgQueryOut)] + [getattr(KsgQueryOut, f).offset for f in QUERY_FIELDS] + [qr.ALLOCATED, qr.OBSERVED, qr.INTERPOLATED, qr.GRADIENT]
    assert got == want
