"""The incremental ESDF rule (csrc/ksg_esdf.cuh, modelled by tests/esdf_incremental_ref.py) equals the batch twin (tests/esdf_ref.py) bit
for bit after every update of edit sequences - random block edits of sphere and plane fields, blocks added, an edit that flips a site
only in the neighbour block, and a site change exactly Rb and Rb + 1 blocks from the output - at voxels_per_side 1, 2, 8 and 16, with
the window W a multiple of voxels_per_side and not.  Two mutants of the rule (dilation by Rb - 1, no face-neighbour site recompute) each
make some case differ, so the scenes are sharp.  And the ESDF point-query twin stays within the bound of ksg_esdf.cuh on a plane."""
import math

import numpy as np
import pytest

import esdf_incremental_ref as ir
import esdf_ref as er
import mesh_ref as mr

F = np.float32
VS = 0.125   # exact in binary: W = ceil(m / vs) + 1 is exactly what the test intends


def _take(exp, keep):
    return {k: np.ascontiguousarray(v[keep]) for k, v in exp.items()}


def _concat(a, b):
    return {k: np.concatenate([a[k], b[k]]) for k in a}


def _differs(state, exp, vps, m):
    """blocks whose stored output is not the batch twin's, bit for bit"""
    want = er.esdf(exp, VS, vps, m)
    bad = []
    for i, b in enumerate(want["block_index"].tolist()):
        d, f = state["out"][tuple(b)]
        if (d.view(np.uint32) != want["distance"][i].view(np.uint32)).any() or (f != want["flags"][i]).any():
            bad.append(tuple(b))
    return bad


def _random_sequence(vps, shape, seed, steps=6):
    """(export, changed blocks) per step: a sphere or plane field over a box of blocks, 60 % of them allocated at first; each step
    edits 1-2 allocated blocks (distance noise, unobserved voxels, or another sphere) and allocates 0-2 more"""
    n = {1: 10, 2: 6, 8: 3, 16: 2}[vps]
    ext = n * vps * VS
    if shape == "sphere":
        fn = lambda x, y, z: np.sqrt(x * x + y * y + z * z) - F(0.3 * ext)                  # noqa: E731
    else:
        fn = lambda x, y, z: F(0.6) * x + F(0.3) * y + F(0.742) * z - F(0.05)              # noqa: E731
    full = mr.sdf_export(fn, VS, vps, -n // 2, n - n // 2)
    rng = np.random.default_rng(seed)
    on = rng.random(len(full["block_index"])) < 0.6
    on[0] = True
    cur = _take(full, on)
    yield cur, []
    V = vps ** 3
    for _ in range(steps):
        cur = {k: v.copy() for k, v in cur.items()}
        nb = len(cur["block_index"])
        changed = []
        for i in rng.choice(nb, size=min(nb, int(rng.integers(1, 3))), replace=False):
            kind = rng.integers(0, 3)
            if kind == 0:
                sel = rng.random(V) < 0.3
                cur["tsdf_distance"][i, sel] += rng.normal(0, 2 * VS, int(sel.sum())).astype(F)
            elif kind == 1:
                cur["tsdf_weight"][i, rng.random(V) < 0.2] = 0.0
            else:
                b = cur["block_index"][i].astype(np.int64)
                lin = np.arange(V)
                g = b * vps + np.stack([lin % vps, (lin // vps) % vps, lin // (vps * vps)], 1)
                c = ((g + 0.5) * VS).astype(F)
                r = F(rng.uniform(0.1, 0.4) * ext)
                cur["tsdf_distance"][i] = np.sqrt((c * c).sum(1)) - r
            changed.append(tuple(cur["block_index"][i].tolist()))
        off = np.flatnonzero(~on)
        if len(off):
            add = rng.choice(off, size=min(len(off), int(rng.integers(0, 3))), replace=False)
            on[add] = True
            cur = _concat(cur, _take(full, add))
        yield cur, changed


def _run(seq, vps, m, **mutant):
    """(blocks that differed from the batch twin over the sequence, the stats of every update)"""
    state, bad, stats = None, 0, []
    for exp, changed in seq:
        state, st = ir.update(state, exp, changed, VS, vps, m, **mutant)
        bad += len(_differs(state, exp, vps, m))
        stats.append(st)
    return bad, stats


def _windows(vps):
    """max_distance values giving a window W that is a multiple of vps, and one that is not (vps > 1)"""
    ws = {1: (3,), 2: (4, 5), 8: (8, 10), 16: (16, 10)}[vps]
    return [(w - 1) * VS for w in ws]


CASES = [(vps, m) for vps in (1, 2, 8, 16) for m in _windows(vps)]


@pytest.mark.parametrize("vps,m", CASES)
@pytest.mark.parametrize("shape", ["sphere", "plane"])
def test_random_edit_sequences_equal_the_batch_twin(vps, m, shape):
    W = er.window(VS, m)
    assert W == round(m / VS) + 1
    bad, stats = _run(list(_random_sequence(vps, shape, 7 * vps + len(shape))), vps, m)
    assert bad == 0
    assert stats[0]["full"] == 1 and all(s["full"] == 0 for s in stats[1:])
    assert all(s["z_blocks"] <= s["blocks"] and s["changed_blocks"] <= s["site_blocks"] for s in stats)


def test_sparse_scenes_rewrite_fewer_blocks_than_the_map():
    """at vps 2 and 8 the box holds blocks beyond Rb of every edit: D is strictly smaller than the map in some update"""
    for vps in (2, 8):
        m = _windows(vps)[0]
        _, stats = _run(list(_random_sequence(vps, "plane", 11, steps=8)), vps, m)
        assert any(s["z_blocks"] < s["blocks"] and s["site_changed"] > 0 for s in stats[1:]), stats


def _face_flip_scene(vps):
    """a plane between blocks 0 and 1 along x whose sites all lie in block 1; the edit makes one voxel of block 0 unobserved, which
    removes the site of block 1 across the face and changes no site byte of block 0"""
    x0 = F(vps * VS + 0.1 * VS)
    exp = mr.sdf_export(lambda x, y, z: x - x0, VS, vps, 0, 2)
    before = ir.sites_by_block(exp, vps)
    edit = {k: v.copy() for k, v in exp.items()}
    i = int(np.flatnonzero(np.all(edit["block_index"] == (0, 0, 0), axis=1))[0])
    edit["tsdf_weight"][i, vps - 1] = 0.0                                  # local (vps - 1, 0, 0): face voxel of block 0
    after = ir.sites_by_block(edit, vps)
    assert (before[(0, 0, 0)] == after[(0, 0, 0)]).all() and not before[(0, 0, 0)].any()
    assert (before[(1, 0, 0)] != after[(1, 0, 0)]).sum() == 1
    return [(exp, []), (edit, [(0, 0, 0)])]


def _reaches(vps, m):
    """whether a site change can move an output exactly Rb blocks away: its nearest voxel there is (Rb - 1) vps + 1 voxels off, and an
    output is below max_distance only for sqrt(Q) < m / vs <= W - 1, so offsets up to W - 2 count (Rb = ceil(W / vps) is conservative)"""
    W, Rb = er.window(VS, m), ir.block_radius(VS, vps, m)
    return (Rb - 1) * vps + 1 <= W - 2


def _radius_scene(vps, m):
    """a row of Rb + 3 blocks along x with no site; the edit puts sites on block 0's +x face.  Block Rb + 1 (Rb vps + 1 > W voxels away)
    does not change; block Rb does where _reaches() says so"""
    Rb = ir.block_radius(VS, vps, m)
    row = [mr.sdf_export(lambda x, y, z: np.ones_like(x), VS, vps, 0, 1) for _ in range(Rb + 3)]
    for i, e in enumerate(row):
        e["block_index"] = e["block_index"] + np.array([i, 0, 0], np.int32)
    exp = row[0]
    for e in row[1:]:
        exp = _concat(exp, e)
    edit = {k: v.copy() for k, v in exp.items()}
    lin = np.arange(vps ** 3)
    edit["tsdf_distance"][0, lin % vps == vps - 1] = F(-0.5 * VS)
    a, b = er.esdf(exp, VS, vps, m), er.esdf(edit, VS, vps, m)
    moved = [(a["distance"][k].view(np.uint32) != b["distance"][k].view(np.uint32)).any() for k in range(Rb + 3)]
    assert moved[Rb] == _reaches(vps, m) and not moved[Rb + 1], moved
    return [(exp, []), (edit, [(0, 0, 0)])], Rb


@pytest.mark.parametrize("vps,m", CASES)
def test_sharp_scenes_equal_the_batch_twin_and_catch_both_mutants(vps, m):
    flip = _face_flip_scene(vps)
    bad, stats = _run(flip, vps, m)
    assert bad == 0 and stats[1]["site_changed"] == 1 and stats[1]["site_blocks"] == 4   # block 0 and its 3 face neighbours
    assert _run(flip, vps, m, face_neighbours=False)[0] > 0
    radius, Rb = _radius_scene(vps, m)
    bad, stats = _run(radius, vps, m)
    assert bad == 0
    assert stats[1]["z_blocks"] == Rb + 1 < stats[1]["blocks"]                   # blocks 0 .. Rb: exactly Rb from the site, not Rb + 1
    assert (_run(radius, vps, m, dilation=Rb - 1)[0] > 0) == _reaches(vps, m)


def test_the_dilation_mutant_is_caught_somewhere():
    assert [c for c in CASES if _reaches(*c)] == [(8, 0.875), (16, 1.875), (16, 1.125)]


def test_the_esdf_query_twin_on_a_plane_is_within_the_bound_of_the_header():
    """trilinear ESDF distance and gradient of an oblique plane's field against the exact distance.  The plane's distance is linear, so
    its trilinear interpolation is exact and the voxel bound of ksg_esdf.cuh carries over: -vs / 2 - 2^-22 m <= D_esdf - D <= sqrt(3) vs
    + 2^-22 m; a central difference of two such values is off by at most (sqrt(3) + 1 / 2) / 2 per component."""
    vps, m = 8, 4.0
    nrm = np.array([0.6, 0.3, 0.742], np.float64)
    nrm /= np.linalg.norm(nrm)
    fn = lambda x, y, z: (F(nrm[0]) * x + F(nrm[1]) * y + F(nrm[2]) * z - F(0.05)).astype(F)   # noqa: E731
    exp = mr.sdf_export(fn, VS, vps, -1, 2)
    state, _ = ir.update(None, exp, [], VS, vps, m)
    layer = ir.as_export(state)
    assert not (layer["flags"] & er.CAPPED).any()
    rng = np.random.default_rng(3)
    p = rng.uniform(-vps * VS, 2 * vps * VS, (4000, 3)).astype(F)
    q = ir.esdf_query(layer, VS, vps, p)
    true = p.astype(np.float64) @ nrm - 0.05
    # the bound needs the surface point nearest p inside the map (beyond its edge there are no sites)
    foot = p.astype(np.float64) - true[:, None] * nrm
    inside = np.all((foot > -vps * VS + 2 * VS) & (foot < 2 * vps * VS - 2 * VS), axis=1)
    ok = ((q["flags"] & 4) != 0) & inside
    assert ok.sum() > 1000
    err = q["distance"][ok].astype(np.float64) - true[ok]
    eps = 2.0 ** -22 * m + 1e-6
    assert err.min() >= -VS / 2 - eps and err.max() <= math.sqrt(3) * VS + eps, (err.min(), err.max())
    g = ((q["flags"] & 8) != 0) & inside
    assert g.sum() > 1000
    gerr = np.abs(q["gradient"][g].astype(np.float64) - nrm).max()
    assert gerr <= (math.sqrt(3) + 0.5) / 2 + 1e-5, gerr
    print(f"distance error {err.min():.4f} .. {err.max():.4f} m, gradient error <= {gerr:.4f}")
