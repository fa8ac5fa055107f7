"""CPU twin (numpy float32, same operation order) of ksg_query_points / csrc/ksg_query.cuh: the containing voxel of each point, voxblox's
trilinear TSDF distance and its central-difference gradient, evaluated on an export dict (like tests/mesh_ref.py).  Restates voxblox's
Interpolator, which is not part of the reference tree - see the header of csrc/ksg_query.cuh.  Test infrastructure."""
import numpy as np

F = np.float32
NAN_BITS = 0x7FC00000
ALLOCATED, OBSERVED, INTERPOLATED, GRADIENT = 1, 2, 4, 8
_BIAS = 1 << 20


def nan(shape):
    """the NaN the kernel writes where a value is not valid"""
    return np.full(shape, NAN_BITS, np.uint32).view(F)


def _pack(b):
    return ((b[:, 2] + _BIAS) << 42) | ((b[:, 1] + _BIAS) << 21) | (b[:, 0] + _BIAS)


def _key_in_range(b):
    return np.all((b >= -_BIAS) & (b < _BIAS), axis=1)


class _Map:
    def __init__(self, exp, voxel_size, vps, min_weight):
        self.vs = F(voxel_size)
        self.vsi = F(1.0 / float(self.vs))          # DevCfg.vsi
        self.vps = vps
        self.vps_inv = F(1.0) / F(vps)              # DevCfg.vps_inv
        self.mw = F(min_weight)
        bi = np.asarray(exp["block_index"], np.int64).reshape(-1, 3)
        keys = _pack(bi)
        self.order = np.argsort(keys, kind="stable")
        self.sorted = keys[self.order]
        self.D = np.asarray(exp["tsdf_distance"], F).reshape(len(bi), -1)
        self.W = np.asarray(exp["tsdf_weight"], F).reshape(len(bi), -1)

    def in_range(self, p):
        """index_in_range(p / vs); False for every non-finite point"""
        with np.errstate(invalid="ignore", over="ignore"):
            return np.all(np.abs(p * self.vsi) < F(1.0e9), axis=1)

    def grid_index(self, p):
        return np.floor(p * self.vsi + F(1e-6)).astype(np.int64)

    def block_of_voxel(self, g):
        return np.floor(g.astype(F) * self.vps_inv).astype(np.int64)

    def voxel(self, g):
        """(block row or -1, linear voxel index) of global voxel indices g [m, 3]"""
        b = self.block_of_voxel(g)
        ok = _key_in_range(b)
        row = np.full(len(g), -1, np.int64)
        if len(self.sorted):
            k = _pack(np.where(ok[:, None], b, 0))
            pos = np.minimum(np.searchsorted(self.sorted, k), len(self.sorted) - 1)
            hit = ok & (self.sorted[pos] == k)
            row = np.where(hit, self.order[pos], -1)
        l = g & (self.vps - 1)
        return row, l[:, 0] + self.vps * (l[:, 1] + self.vps * l[:, 2])

    def interp(self, p):
        """(valid [m], D [m]) trilinear distance over the 8 surrounding voxel centres, all allocated and observed"""
        vs, vsi = self.vs, self.vsi
        ok = self.in_range(p)
        p = np.where(ok[:, None], p, F(0))
        g0 = self.grid_index(p)
        g0 = g0 - (p < (g0.astype(F) + F(0.5)) * vs)
        q = (p - (g0.astype(F) + F(0.5)) * vs) * vsi
        d = np.zeros((len(p), 8), F)
        for i in range(8):
            row, lin = self.voxel(g0 + np.array([i >> 2, (i >> 1) & 1, i & 1], np.int64))
            have = row >= 0
            r = np.where(have, row, 0)
            ok &= have & (self.W[r, lin] > self.mw)
            d[:, i] = self.D[r, lin]
        d0, d1, d2, d3, d4, d5, d6, d7 = (d[:, i] for i in range(8))
        x, y, z = q[:, 0], q[:, 1], q[:, 2]
        b0 = d0
        b1 = -d0 + d4
        b2 = -d0 + d2
        b3 = -d0 + d1
        b4 = ((d0 - d2) - d4) + d6
        b5 = ((d0 - d1) - d2) + d3
        b6 = ((d0 - d1) - d4) + d5
        b7 = ((((((-d0 + d1) + d2) - d3) + d4) - d5) - d6) + d7
        with np.errstate(invalid="ignore", over="ignore"):
            v = ((((((b0 + x * b1) + y * b2) + z * b3) + (x * y) * b4) + (y * z) * b5) + (z * x) * b6) + ((x * y) * z) * b7
        return ok, v.astype(F)


def query(exp, voxel_size, vps, xyz, min_weight=1e-4):
    """exp: export dict (block_index, tsdf_distance, tsdf_weight, tsdf_rgba, sem_label, sem_rgba, optional sem_priors); xyz [n, 3].
    -> dict with the keys and layout of Integrator.query_points()"""
    m = _Map(exp, voxel_size, vps, min_weight)
    p = np.ascontiguousarray(xyz, F).reshape(-1, 3)
    n = len(p)
    valid = m.in_range(p)
    ps = np.where(valid[:, None], p, F(0))
    g = m.grid_index(ps)
    valid &= _key_in_range(m.block_of_voxel(g))
    row, lin = m.voxel(g)
    alloc = valid & (row >= 0)
    r = np.where(alloc, row, 0)
    wgt = m.W[r, lin]
    observed = alloc & (wgt > m.mw)
    out = {"flags": (alloc * ALLOCATED | observed * OBSERVED).astype(np.uint8),
           "tsdf_distance": np.where(alloc, m.D[r, lin], nan(n)),
           "tsdf_weight": np.where(alloc, wgt, nan(n))}
    V = vps ** 3

    def field(k, tail, dt):          # [max(nb, 1), V, *tail]; a field the export lacks reads as zeros
        a = np.asarray(exp[k], dt) if k in exp else np.zeros((len(m.D), V) + tail, dt)
        a = a.reshape((-1, V) + tail)
        return a if len(a) else np.zeros((1, V) + tail, dt)
    for k in ("tsdf_rgba", "sem_rgba"):
        out[k] = np.where(alloc[:, None], field(k, (4,), np.uint8)[r, lin], 0).astype(np.uint8)
    out["sem_label"] = np.where(alloc, field("sem_label", (), np.uint8)[r, lin], 0).astype(np.uint8)
    if "sem_priors" in exp:
        C = np.asarray(exp["sem_priors"]).shape[-1]
        out["sem_priors"] = np.where(alloc[:, None], field("sem_priors", (C,), F)[r, lin], nan((n, C)))
    ok0, d = m.interp(ps)
    ok0 &= valid
    out["flags"] |= (ok0 * INTERPOLATED).astype(np.uint8)
    out["distance"] = np.where(ok0, d, nan(n))
    okg = valid.copy()
    grad = np.zeros((n, 3), F)
    for a in range(3):
        pp, pm = ps.copy(), ps.copy()
        pp[:, a] = ps[:, a] + m.vs
        pm[:, a] = ps[:, a] - m.vs
        okp, dp = m.interp(pp)
        okm, dm = m.interp(pm)
        okg &= okp & okm
        with np.errstate(invalid="ignore", over="ignore"):
            grad[:, a] = (dp - dm) / (F(2.0) * m.vs)
    out["flags"] |= (okg * GRADIENT).astype(np.uint8)
    out["gradient"] = np.where(okg[:, None], grad, nan((n, 3)))
    return out
