"""Numpy model of the device mesh layer's dirty-set rule (ksg_update_mesh, csrc/ksg_mesh.cuh):
  C = blocks stamped since the last update + blocks allocated since it,
  R = allocated blocks b with b + e in C for some e in {0,1}^3 (C and its allocated lower neighbours),
the full-update rule (first update, new min_weight, a block beyond the window bound), and the layer itself: per block, the mesh
mesh_ref.extract gives it, re-meshed for R and kept for every other block.  `rule` selects the exact rule or one of its mutants, which
the CPU test must catch.  Test infrastructure."""
import numpy as np

import mesh_ref

NEAR_VOXELS = 1 << 18          # kMeshNearVoxels
LOWER = [(-(e & 1), -((e >> 1) & 1), -(e >> 2)) for e in range(8)]
RULES = {
    "exact": LOWER,
    "face": [(0, 0, 0), (-1, 0, 0), (0, -1, 0), (0, 0, -1)],        # mutant: face neighbours only
    "upper": [(-a, -b, -c) for a, b, c in LOWER],                    # mutant: upper instead of lower neighbours
}


def far(block, vps):
    """the block lies beyond the window bound: (|b| + 1) * vps + 2 > 2^18 on some axis"""
    return any((abs(int(c)) + 1) * vps + 2 > NEAR_VOXELS for c in block)


def dirty_sets(keys, prev_keys, stamped, rule="exact"):
    """C and R (sets of block tuples).  keys: the blocks now; prev_keys: the blocks at the last update (None: full); stamped: blocks
    stamped since.  rule "no_new" is the mutant that ignores new blocks (stamped or not)."""
    new = set(keys) if prev_keys is None else set(keys) - set(prev_keys)
    C = (set(stamped) & set(keys)) - new if rule == "no_new" else (set(stamped) & set(keys)) | new
    if prev_keys is None:
        C = set(keys)
    offs = RULES["exact" if rule == "no_new" else rule]
    R = {(b[0] + o[0], b[1] + o[1], b[2] + o[2]) for b in C for o in offs} & set(keys)
    return C, R


def split(mesh, block_index=None):
    """{block: (vertices, rgba, labels)} of an extract_mesh-layout dict (block_index: its blocks, when the dict does not list them)"""
    f = mesh["block_first"]
    bidx = mesh["block_index"] if block_index is None else block_index
    return {tuple(int(c) for c in b): (mesh["vertices"][f[i]:f[i + 1]], mesh["rgba"][f[i]:f[i + 1]], mesh["labels"][f[i]:f[i + 1]])
            for i, b in enumerate(np.asarray(bidx).tolist())}


def join(blocks):
    """extract_mesh-layout dict of {block: (vertices, rgba, labels)}, blocks in (z, y, x) order"""
    order = sorted(blocks, key=lambda b: (b[2], b[1], b[0]))
    first = np.zeros(len(order) + 1, np.int64)
    for i, b in enumerate(order):
        first[i + 1] = first[i] + len(blocks[b][0])
    cat = lambda k, shape, dt: np.concatenate([blocks[b][k] for b in order]) if order else np.zeros(shape, dt)   # noqa: E731
    return {"vertices": cat(0, (0, 3), np.float32), "rgba": cat(1, (0, 4), np.uint8), "labels": cat(2, (0,), np.uint8),
            "block_index": np.array(order, np.int32).reshape(-1, 3), "block_first": first}


def update(state, exp, stamped, voxel_size, vps, min_weight=1e-4, rule="exact"):
    """One ksg_update_mesh on the map `exp` (an export dict); stamped = blocks stamped since the last update.  state None = no layer.
    -> (state, stats as ksg_update_mesh reports them).  The layer is state["blocks"]; state["R"] the blocks this update re-meshed."""
    keys = [tuple(int(c) for c in b) for b in exp["block_index"].tolist()]
    full = state is None or state["min_weight"] != min_weight or state["far"]
    if not full and not stamped and set(keys) == set(state["blocks"]):
        st = dict(blocks=len(keys), full=0, changed_blocks=0, remeshed_blocks=0, vertices=state["vertices"], remeshed_vertices=0)
        return dict(state, R=set()), st
    C, R = dirty_sets(keys, None if full else list(state["blocks"]), stamped, rule)
    fresh = split(mesh_ref.extract(exp, voxel_size, vps, min_weight), exp["block_index"]) if keys else {}
    empty = (np.zeros((0, 3), np.float32), np.zeros((0, 4), np.uint8), np.zeros(0, np.uint8))   # what a mutant never meshed
    blocks = {b: (fresh[b] if (b in R or full) else state["blocks"].get(b, empty)) for b in keys}
    new = set(keys) if full else set(keys) - set(state["blocks"])
    now_far = any(far(b, vps) for b in new) or (not full and state["far"])
    vertices = sum(len(v[0]) for v in blocks.values())
    st = dict(blocks=len(keys), full=int(full), changed_blocks=len(C), remeshed_blocks=len(R), vertices=vertices,
              remeshed_vertices=sum(len(blocks[b][0]) for b in R))
    return dict(blocks=blocks, min_weight=min_weight, far=now_far, vertices=vertices, R=R), st


def vertex_window(b, l, oa, ob, vs, vps, sa, sb):
    """One axis of the vertex k_mesh_blocks puts on the cube edge from corner offset oa to ob (0 or 1 each; equal on the axes the edge
    does not run along) of the cube at local index l of block b, with corner distances sa, sb, in the kernel's float32 operation order:
    -> (the containing voxel's index, g = the cube's lower corner's global index).  The window holds when the first is g or g + 1."""
    F = np.float32
    vs = F(vs)
    vsi = F(1.0 / float(vs))
    block_size = F(F(vps) * vs)
    origin = F(F(b) * block_size)
    base = F(origin + F(F(F(l) + F(0.5)) * vs))
    pa = F(base + F(F(oa) * vs))
    pb = F(base + F(F(ob) * vs))
    sa, sb = F(sa), F(sb)
    diff = F(sa - sb)
    if abs(diff) >= F(1e-6):
        t = F(sa / diff)
        p = F(pa + F(t * F(pb - pa)))
    else:
        p = F(F(0.5) * F(pa + pb))
    return int(np.floor(F(F(p * vsi) + F(1e-6)))), b * vps + l
