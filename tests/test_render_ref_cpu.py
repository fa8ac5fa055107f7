"""CPU checks of the render twin (tests/render_ref.py) against independent truth: analytic planes and spheres imported as exports, the
block skip against float64 ray-box crossings, and the synthetic world integrated by the CPU oracle against the noise-free ground truth;
plus the ctypes mirror of ksg_render_out against the C header.  The GPU kernel is compared with this twin bit for bit in
tests/test_gpu_render.py."""
import ctypes as C
import os
import subprocess

import numpy as np

import mesh_ref as mr
import query_ref as qr
import render_ref as rr
from kimera_semantics_b200 import synth
from kimera_semantics_b200.capi import KSG_INTEGRATOR_FAST, RENDER_FIELDS, KsgRenderOut
from oracle.oracle_py import OracleIntegrator
from parity_utils import make_config

F = np.float32
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _rays(T, K, W, H):
    """float64 origin and per-unit-z world directions of the pixels, from the float constants the march uses"""
    cam = rr.Camera(T, K, W, H)
    a = ((cam.fu - cam.cx) * cam.constant_x).astype(np.float64)
    b = ((cam.fv - cam.cy) * cam.constant_y).astype(np.float64)
    w, x, y, z = np.asarray(T, np.float64)[:4]
    R = np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                  [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                  [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])
    d = np.stack([a, b, np.ones_like(a)], 1) @ R.T
    return np.asarray(T, np.float64)[4:], d


def _look_at(eye, target):
    """T_G_C (qw qx qy qz tx ty tz) float32 of a camera at eye whose optical axis (z) points at target"""
    zc = np.asarray(target, np.float64) - eye
    zc /= np.linalg.norm(zc)
    xc = np.cross(zc, [0.0, 0.0, 1.0] if abs(zc[2]) < 0.9 else [1.0, 0.0, 0.0])
    xc /= np.linalg.norm(xc)
    R = np.stack([xc, np.cross(zc, xc), zc], 1)
    w = np.sqrt(max(1e-12, 1 + R[0, 0] + R[1, 1] + R[2, 2])) / 2
    q = np.array([w, (R[2, 1] - R[1, 2]) / (4 * w), (R[0, 2] - R[2, 0]) / (4 * w), (R[1, 0] - R[0, 1]) / (4 * w)])
    return np.concatenate([q / np.linalg.norm(q), eye]).astype(F)


def _slab(o, d, lo, hi):
    """float64 [z_in, z_out] of the rays o + z d inside the box lo..hi (z_in > z_out: no crossing)"""
    with np.errstate(divide="ignore", invalid="ignore"):
        t0, t1 = (lo - o) / d, (hi - o) / d
    return np.nanmax(np.minimum(t0, t1), axis=1), np.nanmin(np.maximum(t0, t1), axis=1)


def test_oblique_plane_depth_is_exact_up_to_rounding():
    vs, vps = 0.1, 8
    n = np.array([0.3, -0.5, 0.81])
    nf = (n / np.linalg.norm(n)).astype(F)
    exp = mr.sdf_export(lambda x, y, z: F(0.3) - (nf[0] * x + nf[1] * y + nf[2] * z), vs, vps, -2, 2)
    T = _look_at(np.array([0.1, -0.2, -1.2]), [0.2, 0.1, 0.3])
    W, H, K = 64, 48, np.array([60.0, 60.0, 31.5, 23.5])
    depth, _ = rr.march(exp, vs, vps, T, K, W, H, 0.1, 3.0)
    o, d = _rays(T, K, W, H)
    nd = nf.astype(np.float64)
    z_true = (np.float64(F(0.3)) - nd @ o) / (d @ nd)
    hit = ~np.isnan(depth)
    p_true = o + z_true[:, None] * d
    inside = (np.abs(p_true) < 2 * vps * vs - vs).all(axis=1) & (z_true > 0.1)    # the crossing lies inside the imported field
    assert inside.mean() > 0.8 and hit[inside].all()
    # trilinear interpolation of a linear field is exact, and so is the linear interpolation between the two samples: what is left is
    # float32 rounding of the sample points and distances, a few ulp at the scene's 2 m scale, measured along the plane's normal
    err = np.abs(depth[hit] - z_true[hit]) * np.abs(d[hit] @ nd)
    assert err.max() <= 4 * np.spacing(F(2.0)), err.max()           # measured 1.6e-7


def _sphere(vs, R, vps=8, blocks=4):
    return mr.sdf_export(lambda x, y, z: np.sqrt(x * x + y * y + z * z) - F(R), vs, vps, -blocks, blocks)


def test_sphere_depth_normals_and_misses():
    """Bound on the depth error.  The sample distances are the trilinear interpolant of |p| - R, whose error is at most
    (vs^2 / 8) * sum_a |d^2f / dx_a^2| <= (vs^2 / 8) * 2 / rho = vs^2 / (4 R) near the surface (rho ~ R).  Seen from outside, |p| is convex
    along the ray, so a step of kappa * D0 (kappa < 1) never crosses the surface: the crossing interval is one minimum step h = vs / 2
    long, and the linear interpolation over it errs by at most (h^2 / 8) * (1 / R) = vs^2 / (32 R) in distance.  A distance error e moves
    the hit by e / cos(theta) along the ray (theta: incidence angle) and by at most that in z (r >= 1).  With R = 20 vs and cos >= 0.2:
    (1/80 + 1/640) vs / 0.2 = 0.070 vs <= 0.1 vs.  The normal is the central difference of the interpolant over 2 vs, whose direction
    errs by O(vs / R): asserted at 2 vs / R rad."""
    vs, R = 0.05, 1.0                                             # R = 20 voxels
    exp = _sphere(vs, R)
    T = _look_at(np.array([0.3, -0.4, -1.45]), [0.05, 0.02, 0.0])
    W, H, K = 48, 40, np.array([24.0, 24.0, 23.5, 19.5])          # wide: the corners miss the sphere
    out = rr.render(exp, vs, 8, T, K, W, H, 0.05, 4.0)
    depth = out["depth"].reshape(-1)
    o, d = _rays(T, K, W, H)
    bq, cq = d @ o, o @ o - R * R
    aq = np.einsum("ij,ij->i", d, d)
    disc = bq * bq - aq * cq
    z_true = (-bq - np.sqrt(np.maximum(disc, 0))) / aq
    p_true = o + z_true[:, None] * d
    cos = -np.einsum("ij,ij->i", p_true / R, d / np.sqrt(aq)[:, None])
    front = (disc > 0) & (cos >= 0.2)
    assert front.sum() > 500 and (disc < 0).sum() > 50
    assert not np.isnan(depth[front]).any()
    assert np.abs(depth[front] - z_true[front]).max() <= 0.1 * vs    # measured 0.012 vs
    # rays that miss the sphere by more than the interpolation error see nothing
    clear = disc < -(0.05 * aq)
    assert clear.sum() > 50 and np.isnan(depth[clear]).all()
    g = out["gradient"].reshape(-1, 3)[front].astype(np.float64)
    assert ((out["flags"].reshape(-1)[front] & qr.GRADIENT) != 0).all()
    nrm = g / np.linalg.norm(g, axis=1, keepdims=True)
    ang = np.arccos(np.clip(np.einsum("ij,ij->i", nrm, p_true[front] / R), -1, 1))
    assert ang.max() <= 2 * vs / R, np.degrees(ang.max())          # 5.7 degrees; measured 0.5
    # every miss carries the query's answer for a NaN point
    miss = np.isnan(depth)
    assert (out["flags"].reshape(-1)[miss] == 0).all() and np.isnan(out["points_G"].reshape(-1, 3)[miss]).all()


def test_camera_inside_the_sphere_renders_no_hit():
    vs = 0.05
    exp = _sphere(vs, 1.0)
    T = _look_at(np.array([0.1, 0.05, -0.2]), [0.3, 0.2, 1.0])
    depth, _ = rr.march(exp, vs, 8, T, np.array([20.0, 20.0, 15.5, 11.5]), 32, 24, 0.05, 4.0)
    assert np.isnan(depth).all()


def test_zero_distance_on_a_sample_is_on_the_non_positive_side():
    vs, vps = 0.125, 8
    exp = mr.sdf_export(lambda x, y, z: F(1.0) - z, vs, vps, -1, 2)
    T, K = np.array([1, 0, 0, 0, 0, 0, 0], F), np.array([100.0, 100.0, 0.0, 0.0])   # one pixel on the optical axis: r = 1
    m = qr._Map(exp, vs, vps, 1e-4)
    ok, d = m.interp(np.array([[0.0, 0.0, 1.0]], F))
    assert ok[0] and d[0] == 0.0
    # the first sample has D = 0: not a hit (no positive predecessor); the next is negative; so a miss
    depth, n = rr.march(exp, vs, vps, T, K, 1, 1, 1.0, 1.5)
    assert np.isnan(depth[0]) and n[0] > 1
    # D0 = vs / 2 at z = 1 - vs / 2, one minimum step lands on D = 0 exactly: the hit, at z = 1 exactly
    depth, n = rr.march(exp, vs, vps, T, K, 1, 1, 1.0 - vs / 2, 1.5)
    assert depth[0] == F(1.0) and n[0] == 2


def test_block_skip_finds_a_plate_in_a_single_block():
    """One allocated block (0, 0, 0) holding a slice of an oblique plane, unallocated space around it.  D(p) is valid in the box V of
    the block's voxel centres.  A ray enters V with a sample at most one voxel past V's entry (it enters the block a quarter voxel past
    the face after a skip, then steps one voxel while D is invalid), and from a positive sample it never steps past the plane by more
    than vs / 2 (a step of kappa * D stops short of a plane).  So every ray that crosses the plane more than one voxel after entering V
    and more than half a voxel before leaving it finds it - also rays that only clip a corner of the block."""
    vs, vps = 0.1, 8
    bs = vs * vps
    n = np.array([0.45, 0.3, -0.84])
    nf = (n / np.linalg.norm(n)).astype(F)
    c = F(nf.astype(np.float64) @ np.array([0.4, 0.4, 0.4]))
    exp = mr.sdf_export(lambda x, y, z: c - (nf[0] * x + nf[1] * y + nf[2] * z), vs, vps, 0, 1)
    rng = np.random.default_rng(5)
    W, H, K = 48, 48, np.array([30.0, 30.0, 23.5, 23.5])           # ~77 degrees: many rays clip edges and corners
    found = corner = 0
    for _ in range(24):
        u = rng.normal(size=3)
        eye = np.array([0.4, 0.4, 0.4]) + u / np.linalg.norm(u) * rng.uniform(0.8, 1.2)
        T = _look_at(eye, np.array([0.4, 0.4, 0.4]) + rng.uniform(-0.3, 0.3, 3))
        depth, _ = rr.march(exp, vs, vps, T, K, W, H, 0.05, 4.0)
        o, d = _rays(T, K, W, H)
        r = np.linalg.norm(d, axis=1)
        z_in, z_out = _slab(o, d, np.full(3, vs / 2), np.full(3, bs - vs / 2))
        nd = nf.astype(np.float64)
        z_c = (np.float64(c) - nd @ o) / (d @ nd)
        toward = (d @ nd) > 0                                      # from the positive side to the negative side
        ok = toward & ((z_c - z_in) * r > 1.0 * vs * 1.001) & ((z_out - z_c) * r > 0.5 * vs * 1.001) & (z_in > 0.05)
        assert not np.isnan(depth[ok]).any(), np.argwhere(ok & np.isnan(depth))[:5]
        if ok.any():
            assert np.abs(depth[ok] - z_c[ok]).max() < 1e-5
        found += ok.sum()
        corner += (ok & ((z_out - z_in) * r < 3 * vs)).sum()
    assert found > 1000 and corner > 20, (found, corner)          # measured 1807 and 41


def test_sampled_blocks_include_every_block_crossed_by_more_than_the_push():
    """Isolated allocated blocks (even indices only, so each is entered from unallocated space) of unobserved voxels (no hit ends a
    ray): every block a ray's [min_depth, max_depth] segment crosses by more than the push (a quarter voxel), computed in float64, is
    among the blocks the ray sampled."""
    vs, vps = 0.1, 4
    bs = vs * vps
    rng = np.random.default_rng(9)
    cand = np.array([(x, y, z) for x in range(-4, 5, 2) for y in range(-4, 5, 2) for z in range(-4, 5, 2)])
    bi = cand[rng.random(len(cand)) < 0.5]
    V = vps ** 3
    exp = {"block_index": bi.astype(np.int32), "tsdf_distance": np.full((len(bi), V), 0.3, F), "tsdf_weight": np.zeros((len(bi), V), F)}
    W, H, K = 24, 24, np.array([14.0, 14.0, 11.5, 11.5])
    checked = 0
    for _ in range(6):
        u = rng.normal(size=3)
        eye = u / np.linalg.norm(u) * rng.uniform(0.5, 2.5)
        T = _look_at(eye, rng.uniform(-1.0, 1.0, 3))
        zmin, zmax = 0.05, 3.0
        depth, _, seen = rr.march(exp, vs, vps, T, K, W, H, zmin, zmax, blocks=True)
        assert np.isnan(depth).all()
        o, d = _rays(T, K, W, H)
        r = np.linalg.norm(d, axis=1)
        got = {tuple(row) for row in seen.tolist()}
        for b in bi:
            z_in, z_out = _slab(o, d, b * bs, (b + 1) * bs)
            z_in, z_out = np.maximum(z_in, zmin), np.minimum(z_out, zmax)
            need = np.nonzero((z_out - z_in) * r > 0.25 * vs * 1.01 + 1e-6)[0]
            checked += len(need)
            missing = [i for i in need if (i, *b) not in got]
            assert not missing, (b, missing[:5])
    assert checked > 200, checked


def _oracle_scene(C=21, W=160, H=120, n=9, vs=0.05):
    cfg = make_config(KSG_INTEGRATOR_FAST, vs, C, max_points=W * H)
    ora = OracleIntegrator(cfg)
    cam = synth.make_camera(W, H)
    for f in range(n):
        depth, label, T = synth.frame(cam, f, C)
        ora.integrate_depth(T, depth, label, cam.K)
    exp = ora.export()
    ora.close()
    return exp, cam, cfg


def _against_truth(exp, cam, cfg, T, C):
    vs, vps = cfg.voxel_size, cfg.voxels_per_side
    K = np.array([cam.fx, cam.fy, cam.cx, cam.cy], np.float64)
    out = rr.render(exp, vs, vps, T, K, cam.width, cam.height, 0.1, 6.0)
    d_true, l_true, _ = synth.frame(cam, 0, C, T_G_C=T, depth_noise=0.0, label_noise=0.0)
    # the true surface point of every pixel, and whether the stream observed it (its trilinear distance exists there)
    o, d = _rays(T, K, cam.width, cam.height)
    z = d_true.reshape(-1).astype(np.float64)
    p = (o + z[:, None] * d).astype(F)
    seen = (qr.query(exp, vs, vps, p)["flags"] & qr.INTERPOLATED) != 0
    depth = out["depth"].reshape(-1)
    hit = ~np.isnan(depth)
    dz = np.abs(depth - z)[seen & hit]
    # labels away from the 0.5 m checker boundaries of the synthetic world (two voxels of margin)
    frac = np.abs(p.astype(np.float64) / 0.5 - np.round(p.astype(np.float64) / 0.5)) * 0.5
    inner = seen & hit & (frac.min(axis=1) > 2 * vs)
    agree = (out["sem_label"].reshape(-1) == l_true.reshape(-1))[inner].mean()
    return (seen & hit).sum() / seen.sum(), np.median(dz), np.percentile(dz, 99), agree, seen.sum(), inner.sum()


def test_synthetic_world_render_matches_the_ground_truth():
    C = 21
    exp, cam, cfg = _oracle_scene(C)
    vs = cfg.voxel_size
    # at an integrated pose and between two: coverage 0.810 / 0.816, median |dz| 0.104 / 0.103 vs, p99 1.87 / 1.27 vs,
    # labels 0.968 / 0.970.  A pixel the stream observed can still miss: the march forgets its positive sample where D(p) has an
    # unobserved corner, and the few frames of this scene leave such gaps just in front of the surface
    for f in (4, 4.5):
        cov, med, p99, agree, n_seen, n_inner = _against_truth(exp, cam, cfg, synth.pose(f), C)
        assert n_seen > 8000 and n_inner > 1000
        assert cov >= 0.75 and med <= 0.2 * vs and p99 <= 2.5 * vs and agree >= 0.95, (f, cov, med / vs, p99 / vs, agree)


def test_render_out_mirror_matches_the_c_header(tmp_path):
    src = tmp_path / "r.c"
    fields = ", ".join(["offsetof(ksg_render_out, depth)", "offsetof(ksg_render_out, points_G)"] +
                       [f"offsetof(ksg_render_out, at_hit.{f})" for f in RENDER_FIELDS[2:]])
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "ksg.h"\nint main(){size_t v[] = {sizeof(ksg_render_out), ' + fields +
                   '}; for (size_t i = 0; i < sizeof(v) / sizeof(v[0]); ++i) printf("%zu ", v[i]); printf("\\n"); return 0;}\n')
    exe = tmp_path / "r"
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    got = [int(x) for x in subprocess.check_output([str(exe)]).split()]
    at = KsgRenderOut.at_hit.offset
    want = ([C.sizeof(KsgRenderOut), KsgRenderOut.depth.offset, KsgRenderOut.points_G.offset] +
            [at + getattr(type(KsgRenderOut().at_hit), f).offset for f in RENDER_FIELDS[2:]])
    assert got == want
