"""The numpy twin of ksg_compute_esdf (tests/esdf_ref.py) against truth that does not come from the twin: scipy's exact Euclidean
distance transform of the surface voxels, a per-voxel site rule read straight from the export, brute-force windows, planes through
voxel centres, and the analytic distance of an oblique plane and a sphere within the bound csrc/ksg_esdf.cuh derives."""
import math

import numpy as np
import pytest
from scipy import ndimage

import esdf_ref as er
import mesh_ref as mr

F = np.float32


def _random_field(vps, seed, blocks, vs):
    """an export of `blocks` with a smooth random field plus noise (many sign changes), about 10 % unobserved voxels"""
    rng = np.random.default_rng(seed)
    V = vps ** 3
    lin = np.arange(V)
    l = np.stack([lin % vps, (lin // vps) % vps, lin // (vps * vps)], 1)
    k = rng.normal(size=(3, 3))
    bi = np.array(blocks, np.int32)
    g = (bi[:, None, :] * vps + l[None]).astype(np.float64) + 0.5
    d = sum(np.sin(g @ k[i] * 0.35 + i) for i in range(3)) * vs * 2 + rng.normal(scale=0.2 * vs, size=g.shape[:2])
    w = rng.choice(np.array([0.0, 1e-4, 1.0, 3.0], F), size=(len(bi), V), p=[0.07, 0.03, 0.6, 0.3])
    return {"block_index": bi, "tsdf_distance": d.astype(F), "tsdf_weight": w}


def _sites_direct(exp, vps, min_weight=1e-4):
    """the site rule voxel by voxel from the export's blocks (dict lookups, no dense grid)"""
    where = {tuple(b): i for i, b in enumerate(exp["block_index"].tolist())}
    V = vps ** 3
    out = np.zeros((len(where), V), bool)
    for i, b in enumerate(exp["block_index"].tolist()):
        for v in range(V):
            l = (v % vps, (v // vps) % vps, v // (vps * vps))
            d, w = exp["tsdf_distance"][i, v], exp["tsdf_weight"][i, v]
            if not w > F(min_weight):
                continue
            for a in range(3):
                for s in (-1, 1):
                    g = [b[k] * vps + l[k] for k in range(3)]
                    g[a] += s
                    j = where.get(tuple(x // vps for x in g))
                    if j is None:
                        continue
                    u = (g[0] % vps) + vps * ((g[1] % vps) + vps * (g[2] % vps))
                    dn, wn = exp["tsdf_distance"][j, u], exp["tsdf_weight"][j, u]
                    if wn > F(min_weight) and (d > 0) != (dn > 0) and abs(d) <= abs(dn):
                        out[i, v] = True
    return out


def _edt_expectation(exp, vps, vs, m):
    """sign * min(m, fl(sqrtf(R) * vs)) with R = round(edt(~site)^2) over the padded grid, and whether it is capped"""
    lo, obs, dist, _ = er.dense(exp, vps)
    site = er.sites(obs, dist)
    R = np.rint(ndimage.distance_transform_edt(~site) ** 2)
    mag = (np.sqrt(R.astype(F)) * F(vs)).astype(F)
    capped = ~(mag < F(m))
    mag = np.where(capped, F(m), mag)
    want = np.where(dist > 0, mag, -mag).astype(F)
    lin = np.arange(vps ** 3)
    l = np.stack([lin % vps, (lin // vps) % vps, lin // (vps * vps)], 1)
    g = exp["block_index"].astype(np.int64)[:, None, :] * vps + l[None] - lo
    at = lambda a: a[g[..., 0], g[..., 1], g[..., 2]]  # noqa: E731
    return at(want), at(capped), at(site)


def _cluster(lo, hi):
    return [(x, y, z) for z in range(lo[2], hi[2]) for y in range(lo[1], hi[1]) for x in range(lo[0], hi[0])]


@pytest.mark.parametrize("vps,m", [(2, 0.375), (2, 0.25), (4, 0.875), (4, 0.5), (8, 0.3), (8, 0.875)])
def test_distance_transform_equals_scipy(vps, m):
    vs = 0.125                                                   # exact in binary: W = m / vs + 1
    W = er.window(vs, m)
    # two clusters of blocks, with unallocated blocks between them, plus a lone block further out
    blocks = _cluster((0, 0, 0), (3, 2, 2)) + _cluster((5, 0, 1), (7, 2, 2)) + [(0, 0, 4)]
    exp = _random_field(vps, vps * 7 + W, blocks, vs)
    got = er.esdf(exp, vs, vps, m)
    want, capped, site = _edt_expectation(exp, vps, vs, m)
    assert (site == _sites_direct(exp, vps)).all()
    obs = exp["tsdf_weight"] > F(1e-4)
    plain = obs & ~site
    assert plain.sum() > 50 and site.sum() > 10
    assert (got["distance"][plain].view(np.uint32) == want[plain].view(np.uint32)).all()
    assert (got["flags"][plain] == np.where(capped[plain], er.OBSERVED | er.CAPPED, er.OBSERVED)).all()
    assert (got["flags"][site] == er.OBSERVED | er.SURFACE).all()
    assert (got["distance"][site].view(np.uint32) == exp["tsdf_distance"][site].view(np.uint32)).all()
    assert not capped[plain].all()
    # W is a multiple of vps for half of the parameters
    assert (W % vps == 0) == (m in (0.375, 0.875))


def test_sites_several_unallocated_blocks_away_reach_the_output():
    vps, vs, m = 2, 0.125, 1.5
    blocks = _cluster((0, 0, 0), (2, 2, 2)) + _cluster((5, 0, 0), (6, 1, 1))     # three unallocated blocks (6 voxels) between
    exp = _random_field(vps, 3, blocks, vs)
    far = exp["block_index"][:, 0] == 5
    exp["tsdf_distance"][far] = F(4 * vs)                                        # the far block holds no site of its own ...
    exp["tsdf_weight"][far] = F(1.0)
    got = er.esdf(exp, vs, vps, m)
    want, capped, site = _edt_expectation(exp, vps, vs, m)
    assert not site[far].any()
    assert not capped[far].all()                                                 # ... and is reached from the sites 6+ voxels away
    assert (got["distance"][far].view(np.uint32) == want[far].view(np.uint32)).all()
    assert (got["flags"][far] == np.where(capped[far], er.OBSERVED | er.CAPPED, er.OBSERVED)).all()


def test_window_of_one_voxel_equals_a_brute_force_window():
    vps, vs, m = 4, 0.125, 10.0
    exp = _random_field(vps, 11, _cluster((0, 0, 0), (2, 2, 1)), vs)
    lo, obs, dist, _ = er.dense(exp, vps)
    site = er.sites(obs, dist)
    Q = er.squared(site, 1)
    brute = np.full(site.shape, er.NONE, np.int64)
    sx, sy, sz = site.shape
    for p in np.argwhere(site):
        for o in np.ndindex(3, 3, 3):
            q = p + np.array(o) - 1
            if (q >= 0).all() and (q < (sx, sy, sz)).all():
                brute[tuple(q)] = min(brute[tuple(q)], int(((np.array(o) - 1) ** 2).sum()))
    assert (Q == brute).all()
    assert {0, 1, 2, 3} <= set(np.unique(Q[Q < er.NONE]).tolist())
    out = er.esdf(exp, vs, vps, m, W=1)
    plain = (out["flags"] & er.OBSERVED).astype(bool) & ~(out["flags"] & er.SURFACE).astype(bool)
    near = plain & ~(out["flags"] & er.CAPPED).astype(bool)
    assert near.any() and (np.isin(np.abs(out["distance"][near]), F(vs) * np.sqrt(np.array([1, 2, 3], F)))).all()


@pytest.mark.parametrize("vps", [4, 8])
def test_axis_aligned_plane_through_voxel_centres(vps):
    vs, m = 0.125, 0.6
    c = F((3 + 0.5) * vs)                                        # the plane x = c passes through the centres of voxel layer 3
    exp = mr.sdf_export(lambda x, y, z: x - c, vs, vps, -1, 2)
    got = er.esdf(exp, vs, vps, m)
    d = exp["tsdf_distance"]
    k = np.rint(d / F(vs)).astype(int)                          # layers away from the plane
    assert (d == k * F(vs)).all()
    assert ((got["flags"] & er.SURFACE) != 0).tolist() == (k == 0).tolist()
    assert (got["distance"][k == 0] == 0).all()
    mag = (np.abs(k) * F(vs)).astype(F)
    inside = (k != 0) & (mag < F(m))
    assert (got["distance"][inside] == np.sign(k[inside]) * mag[inside]).all()
    assert (got["flags"][inside] == er.OBSERVED).all()
    beyond = (k != 0) & ~(mag < F(m))
    assert beyond.any() and (got["distance"][beyond] == np.sign(k[beyond]) * F(m)).all()
    assert (got["flags"][beyond] == er.OBSERVED | er.CAPPED).all()


def _check_bound(exp, vps, vs, m, true_d, margin):
    """the error bound of csrc/ksg_esdf.cuh; returns the measured (min, max) of (out - D) / vs over the checked voxels"""
    got = er.esdf(exp, vs, vps, m)
    fl = got["flags"]
    D = np.abs(true_d)
    d = exp["tsdf_distance"]
    site = (fl & er.SURFACE) != 0
    assert (np.abs(d[site]) <= F(vs) / 2 + 1e-7).all()
    # every sign is right (sites carry their own distance, which may be 0)
    nz = ~site
    assert ((got["distance"][nz] > 0) == (d[nz] > 0)).all()
    eps = 2.0 ** -22 * m + 1e-6
    plain = ~site & ((fl & er.CAPPED) == 0) & margin
    err = got["distance"][plain].astype(np.float64) * np.sign(true_d[plain]) - D[plain]
    assert (err >= -vs / 2 - eps).all() and (err <= math.sqrt(3) * vs + eps).all()
    capped = ((fl & er.CAPPED) != 0) & margin
    assert capped.any() and (D[capped] >= m - math.sqrt(3) * vs - eps).all()
    return err.min() / vs, err.max() / vs


def _centres(exp, vps, vs):
    lin = np.arange(vps ** 3)
    l = np.stack([lin % vps, (lin // vps) % vps, lin // (vps * vps)], 1)
    g = exp["block_index"].astype(np.int64)[:, None, :] * vps + l[None]
    return (g + 0.5) * vs


def test_oblique_plane_and_sphere_within_the_derived_bound():
    vps, vs, m = 8, 0.05, 0.4
    lo, hi = -2, 2
    # the grid spans [-0.8, 0.8); only voxels whose ball of radius D + 2 voxels lies inside it are checked (the nearest surface point
    # and its cell must be in the grid)
    n = np.array([0.48, -0.6, 0.64])
    n = n / np.linalg.norm(n)
    off = 0.5 * vs * 0.37
    exp = mr.sdf_export(lambda x, y, z: (n[0] * x + n[1] * y + n[2] * z - off).astype(F), vs, vps, lo, hi)
    p = _centres(exp, vps, vs)
    true_d = p @ n - off
    room = np.min(np.minimum(p - lo * vps * vs, hi * vps * vs - p), axis=-1)
    plane = _check_bound(exp, vps, vs, m, true_d, room > np.abs(true_d) + 2 * vs)
    # the bound is -0.5 .. +1.73 voxel (plus rounding); measured here: -0.312 .. +0.675
    assert plane[0] < -0.3 and plane[1] > 0.6, plane

    R, c = 20 * vs, np.array([0.013, -0.021, 0.007])
    exp = mr.sdf_export(lambda x, y, z: (np.sqrt((x - c[0]) ** 2 + (y - c[1]) ** 2 + (z - c[2]) ** 2) - R).astype(F), vs, vps, -3, 3)
    p = _centres(exp, vps, vs)
    true_d = np.linalg.norm(p - c, axis=-1) - R
    room = np.min(np.minimum(p + 3 * vps * vs, 3 * vps * vs - p), axis=-1)
    sphere = _check_bound(exp, vps, vs, m, true_d, room > np.abs(true_d) + 2 * vs)
    # the bound is -0.5 .. +1.73 voxel (plus rounding); measured here: -0.481 .. +0.689
    assert sphere[0] < -0.4 and sphere[1] > 0.6, sphere


def test_a_site_just_beyond_max_distance_caps_and_a_wider_window_changes_nothing():
    vps, vs = 4, 0.125
    for m in (1.0, 0.99):                                        # W = 9 either way; 8 layers = 1.0 m, not < m
        exp = mr.sdf_export(lambda x, y, z: x - F(0.5 * vs), vs, vps, 0, 3)   # sites: the layer x = 0
        got = er.esdf(exp, vs, vps, m)
        lx = (np.arange(vps ** 3) % vps)[None, :] + exp["block_index"][:, :1] * vps
        assert (got["flags"][lx == 8] == er.OBSERVED | er.CAPPED).all() and (got["distance"][lx == 8] == F(m)).all()
        assert (got["flags"][lx == 7] == er.OBSERVED).all() and (got["distance"][lx == 7] == F(7 * vs)).all()
        wide = er.esdf(exp, vs, vps, m, W=2 * er.window(vs, m))
        assert all(got[k].tobytes() == wide[k].tobytes() for k in got)
    exp = _random_field(2, 5, _cluster((0, 0, 0), (6, 5, 4)), vs)
    for m in (0.25, 0.6):
        a, b = er.esdf(exp, vs, 2, m), er.esdf(exp, vs, 2, m, W=2 * er.window(vs, m))
        assert all(a[k].tobytes() == b[k].tobytes() for k in a)
        assert ((a["flags"] & er.CAPPED) != 0).any()


def test_unobserved_voxels_are_nan_with_no_flags():
    vps, vs = 4, 0.125
    exp = _random_field(vps, 2, _cluster((0, 0, 0), (3, 2, 1)), vs)
    exp["tsdf_weight"][1] = 0.0                                  # a block with no observed voxel
    got = er.esdf(exp, vs, vps, 0.5)
    un = ~(exp["tsdf_weight"] > F(1e-4))
    assert un[1].all() and un[0].any()
    assert (got["distance"][un].view(np.uint32) == er.NAN_BITS).all()
    assert (got["flags"][un] == 0).all()
    assert (got["flags"][~un] & er.OBSERVED).all()
    empty = er.esdf({"block_index": np.zeros((0, 3), np.int32), "tsdf_distance": np.zeros((0, 64), F),
                     "tsdf_weight": np.zeros((0, 64), F)}, vs, vps, 0.5)
    assert empty["distance"].shape == (0, 64) and empty["flags"].shape == (0, 64)
