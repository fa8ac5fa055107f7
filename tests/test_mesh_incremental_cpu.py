"""CPU checks of the device mesh layer's dirty-set rule (csrc/ksg_mesh.cuh, tests/mesh_incremental_ref.py): on random edit sequences
- single voxels at block corners, edges and faces, weights crossing min_weight, new blocks - re-meshing R with mesh_ref.extract and
keeping every other block's mesh equals mesh_ref.extract of the edited map bit for bit; each mutant of the rule (face neighbours only,
upper instead of lower neighbours, new blocks ignored) fails on some sequence; and the window bound that the rule relies on holds at
K = 2^18 and fails far out."""
import itertools

import numpy as np
import pytest

import mesh_incremental_ref as ir
import mesh_ref

F = np.float32
VS, VPS, MW = 0.1, 4, 1e-4


def _start(rng):
    """a 3 x 3 x 3 block map of a sphere's signed distance, with some unobserved voxels"""
    exp = mesh_ref.sdf_export(lambda x, y, z: np.sqrt((x - 0.61) ** 2 + (y - 0.58) ** 2 + (z - 0.63) ** 2) - F(0.45), VS, VPS, 0, 3)
    exp["tsdf_weight"][rng.random(exp["tsdf_weight"].shape) < 0.05] = 0.0
    return exp


def _edit(exp, rng):
    """one edit; returns (the edited export, the block it stamped)"""
    nb = len(exp["block_index"])
    kind = rng.integers(4)
    if kind == 3:                                                     # a new block next to the map, with its own voxels
        while True:
            b = tuple(int(c) for c in rng.integers(-1, 4, 3))
            if b not in {tuple(x) for x in exp["block_index"].tolist()}:
                break
        V = VPS ** 3
        new = {"block_index": np.array([b], np.int32), "tsdf_distance": rng.normal(0, VS, (1, V)).astype(F),
               "tsdf_weight": np.full((1, V), 1.0, F), "tsdf_rgba": rng.integers(0, 256, (1, V, 4)).astype(np.uint8),
               "sem_label": rng.integers(0, 20, (1, V)).astype(np.uint8)}
        exp = {k: np.concatenate([exp[k], new[k]]) for k in exp}
        order = np.lexsort(exp["block_index"].T)                      # keys (z, y, x) as the export lists them
        return {k: v[order] for k, v in exp.items()}, b
    i = int(rng.integers(nb))
    lo, hi = 0, VPS - 1
    pick = lambda: int(rng.choice([lo, hi]))                          # noqa: E731
    mid = lambda: int(rng.integers(VPS))                              # noqa: E731
    lx, ly, lz = [(pick(), pick(), pick()), (pick(), pick(), mid()), (pick(), mid(), mid())][kind]   # corner, edge, face voxel
    lx, ly, lz = rng.permutation([lx, ly, lz])
    v = int(lx + VPS * (ly + VPS * lz))
    exp = {k: a.copy() for k, a in exp.items()}
    if rng.random() < 0.5:
        exp["tsdf_distance"][i, v] = F(-exp["tsdf_distance"][i, v] if exp["tsdf_distance"][i, v] != 0 else VS)
    else:                                                             # weight crossing min_weight, either way
        exp["tsdf_weight"][i, v] = F(0.0) if exp["tsdf_weight"][i, v] > MW else F(1.0)
    exp["tsdf_rgba"][i, v] = rng.integers(0, 256, 4)
    exp["sem_label"][i, v] = rng.integers(0, 20)
    return exp, tuple(int(c) for c in exp["block_index"][i])


def _batch(exp):
    return dict(mesh_ref.extract(exp, VS, VPS, MW), block_index=exp["block_index"])


def _same(a, b):
    return all(a[k].shape == b[k].shape and a[k].tobytes() == b[k].tobytes() for k in ("vertices", "rgba", "labels", "block_index", "block_first"))


def _run(seed, rule, steps=6, edits=3):
    """True when the layer equals the batch mesh after every update of the sequence"""
    rng = np.random.default_rng(seed)
    exp = _start(rng)
    state, _ = ir.update(None, exp, set(), VS, VPS, MW, rule)
    for _ in range(steps):
        stamped = set()
        for _ in range(int(rng.integers(1, edits + 1))):
            exp, b = _edit(exp, rng)
            stamped.add(b)
        state, st = ir.update(state, exp, stamped, VS, VPS, MW, rule)
        if not _same(ir.join(state["blocks"]), _batch(exp)):
            return False
    return True


def test_the_rule_is_exact_on_random_edits():
    assert all(_run(seed, "exact") for seed in range(8))


@pytest.mark.parametrize("rule", ["face", "upper", "no_new"])
def test_each_mutant_fails_on_some_sequence(rule):
    assert not all(_run(seed, rule) for seed in range(8)), rule


def test_a_corner_voxel_reaches_the_diagonal_lower_neighbour():
    """voxel (0, 0, 0) of block (1, 1, 1) is a cube corner of block (0, 0, 0) only: exact re-meshes it, face-only does not"""
    exp = _start(np.random.default_rng(1))
    state, _ = ir.update(None, exp, set(), VS, VPS, MW)
    i = [tuple(b) for b in exp["block_index"].tolist()].index((1, 1, 1))
    before = ir.split(_batch(exp))[(0, 0, 0)]
    e2 = {k: v.copy() for k, v in exp.items()}
    e2["tsdf_distance"][i, 0] = -e2["tsdf_distance"][i, 0] if e2["tsdf_distance"][i, 0] != 0 else F(-VS)
    e2["tsdf_weight"][i, 0] = 1.0
    after = ir.split(_batch(e2))[(0, 0, 0)]
    assert before[0].tobytes() != after[0].tobytes()
    _, R = ir.dirty_sets([tuple(b) for b in e2["block_index"].tolist()], [tuple(b) for b in exp["block_index"].tolist()], {(1, 1, 1)})
    _, R_face = ir.dirty_sets([tuple(b) for b in e2["block_index"].tolist()], [tuple(b) for b in exp["block_index"].tolist()], {(1, 1, 1)}, "face")
    assert (0, 0, 0) in R and (0, 0, 0) not in R_face
    st, stats = ir.update(state, e2, {(1, 1, 1)}, VS, VPS, MW)
    assert stats["full"] == 0 and stats["changed_blocks"] == 1 and stats["remeshed_blocks"] == 8
    assert _same(ir.join(st["blocks"]), _batch(e2))


def _edge_cases(rng, n=64):
    """corner distances of a crossed edge: t at 0, at 1, tiny and huge magnitudes, the midpoint branch, and random ones"""
    fixed = [(0.0, -1.0), (-1.0, 0.0), (1e-7, -1e-7), (-3e-7, 2e-7), (1.0, -1e-30), (-1e-30, 1.0), (0.5, -0.5), (-1e-3, 1e3), (1e3, -1e-3)]
    r = rng.random((n, 2)).astype(F) * F(2.0)
    return fixed + [(float(a), -float(b)) for a, b in r] + [(-float(a), float(b)) for a, b in r]


@pytest.mark.parametrize("vps", [1, 8, 16, 64])
def test_the_window_holds_up_to_the_bound(vps):
    """every vertex of a cube of a block with K = (|b| + 1) * vps + 2 <= 2^18 has its containing voxel in {g, g + 1} per axis"""
    rng = np.random.default_rng(vps)
    bmax = (ir.NEAR_VOXELS - 2) // vps - 1
    assert not ir.far((bmax, 0, 0), vps) and ir.far((bmax + 1, 0, 0), vps) and ir.far((-bmax - 1, 0, 0), vps)
    for vs in (0.01, 0.02, 0.05, 0.1, 0.3, 1.0 / 3.0, 2.0, 7.77):
        for b in (bmax, -bmax, bmax - 1, -bmax + 1, bmax // 2, 0, -1):
            for l in sorted({0, vps - 1, vps // 2}):
                for oa, ob in ((0, 1), (1, 0), (0, 0), (1, 1)):
                    for sa, sb in _edge_cases(rng, 16):
                        got, g = ir.vertex_window(b, l, oa, ob, vs, vps, sa, sb)
                        assert got in (g, g + 1), (vs, b, l, oa, ob, sa, sb, got, g)


def test_the_window_fails_far_out():
    """far beyond the bound the float32 vertex can land outside {g, g + 1}: the fallback lookup is real there"""
    rng = np.random.default_rng(0)
    bad = 0
    for vs, b, l, (sa, sb) in itertools.product((0.05, 0.1, 0.3), ((1 << 20) - 1, -(1 << 20)), range(0, 64, 3), _edge_cases(rng, 4)):
        got, g = ir.vertex_window(b, l, 0, 1, vs, 64, sa, sb)
        bad += got not in (g, g + 1)
    assert bad > 0
