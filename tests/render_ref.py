"""CPU twin (numpy float32, same operation order) of ksg_render_view / csrc/ksg_render.cuh: per pixel a ray march to the first zero
crossing of the trilinear TSDF distance, then the point query at the hit.  Evaluated on an export dict; D(p) is query_ref's
_Map.interp and the outputs at the hit are query_ref.query, so only the march is restated here.  Vectorised over the rays still
marching.  Test infrastructure."""
import numpy as np

import query_ref as qr

F = np.float32
KAPPA = F(0.9)      # kRenderKappa
PUSH = F(0.25)      # kRenderPush (of a voxel)


def _cross(a, b):
    return np.stack([a[:, 1] * b[:, 2] - a[:, 2] * b[:, 1], a[:, 2] * b[:, 0] - a[:, 0] * b[:, 2], a[:, 0] * b[:, 1] - a[:, 1] * b[:, 0]], 1)


def xform_apply(T, p):
    """minkindr QuatTransformation<float> (ksg_device.cuh xform_apply): (p + w*uv + qv x uv) + t with uv = 2*(qv x p)"""
    T = np.asarray(T, F)
    qv = np.broadcast_to(T[1:4], p.shape)
    uv = _cross(qv, p)
    uv = uv + uv
    r = (p + uv * T[0]) + _cross(qv, uv)
    return r + T[4:7]


class Camera:
    """the float constants of one render call, as ksg_render_view derives them from K (float64)"""
    def __init__(self, T, K, width, height):
        K = np.asarray(K, np.float64)
        self.T = np.asarray(T, F)
        self.cx, self.cy = F(K[2]), F(K[3])
        self.constant_x, self.constant_y = F(1.0 / K[0]), F(1.0 / K[1])
        self.W, self.H = width, height
        v, u = np.divmod(np.arange(width * height, dtype=np.int64), width)
        self.fu, self.fv = u.astype(F), v.astype(F)

    def point(self, i, z):
        """p_G(z) of the pixels i"""
        pc = np.stack([((self.fu[i] - self.cx) * z) * self.constant_x, ((self.fv[i] - self.cy) * z) * self.constant_y, z], 1)
        return xform_apply(self.T, pc.astype(F))


def march(exp, voxel_size, vps, T, K, width, height, min_depth, max_depth, min_weight=1e-4, blocks=False, pixels=None):
    """-> (depth [H*W] f32, NaN on a miss, samples per ray [H*W], and with blocks=True the (ray, block x, y, z) rows of every sample's
    containing block, unallocated ones included).  pixels: march only these pixel indices (the others stay NaN with 0 samples)"""
    m = qr._Map(exp, voxel_size, vps, min_weight)
    cam = Camera(T, K, width, height)
    n = width * height
    vs, bs = m.vs, F(vps) * m.vs
    a = (cam.fu - cam.cx) * cam.constant_x
    b = (cam.fv - cam.cy) * cam.constant_y
    r = np.sqrt((a * a + b * b) + F(1)).astype(F)
    Tr = cam.T.copy()
    Tr[4:] = 0
    dirs = xform_apply(Tr, np.stack([a, b, np.ones(n, F)], 1).astype(F))
    step_vox, step_half, step_push = vs / r, (F(0.5) * vs) / r, (PUSH * vs) / r
    z = np.full(n, F(min_depth), F)
    z0 = np.zeros(n, F)
    d0 = np.zeros(n, F)
    pos = np.zeros(n, bool)
    depth = qr.nan(n)
    samples = np.zeros(n, np.int64)
    live = np.arange(n) if pixels is None else np.unique(np.asarray(pixels, np.int64))
    seen = []
    maxd = F(max_depth)
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        while True:
            live = live[z[live] <= maxd]
            if not len(live):
                break
            i = live
            samples[i] += 1
            p = cam.point(i, z[i])
            ok = m.in_range(p)                                                   # (a)
            g = m.grid_index(np.where(ok[:, None], p, F(0)))
            bc = m.block_of_voxel(g)
            ok &= qr._key_in_range(bc)
            if blocks:
                seen.append(np.concatenate([i[ok, None], bc[ok]], 1))
            i, p, g, bc = i[ok], p[ok], g[ok], bc[ok]
            alloc = m.voxel(g)[0] >= 0
            # (b) the ray's exit from the unallocated block, plus the push
            u = ~alloc
            iu, pu, bu, du = i[u], p[u], bc[u], dirs[i[u]]
            t = np.full(len(iu), np.inf, F)
            for ax in range(3):
                hi_face = (bu[:, ax] + 1).astype(F) * bs
                lo_face = bu[:, ax].astype(F) * bs
                face = np.where(du[:, ax] > 0, hi_face, lo_face)
                ta = np.where(du[:, ax] != 0, (face - pu[:, ax]) / du[:, ax], F(np.inf)).astype(F)
                t = np.minimum(t, ta)
            z[iu] = (z[iu] + np.maximum(t, F(0))) + step_push[iu]
            pos[iu] = False
            i, p = i[alloc], p[alloc]
            valid, d = m.interp(p)
            ic = i[~valid]                                                       # (c)
            z[ic] = z[ic] + step_vox[ic]
            pos[ic] = False
            i, d = i[valid], d[valid]
            dp = d > 0                                                           # (d)
            ip, dpos = i[dp], d[dp]
            z0[ip] = z[ip]
            d0[ip] = dpos
            pos[ip] = True
            z[ip] = z[ip] + np.maximum(KAPPA * dpos, F(0.5) * vs) / r[ip]
            i, d = i[~dp], d[~dp]                                                # (e)
            hit = pos[i]
            ih, dh = i[hit], d[hit]
            depth[ih] = z0[ih] + (z[ih] - z0[ih]) * (d0[ih] / (d0[ih] - dh))
            im = i[~hit]
            z[im] = z[im] + step_half[im]
            live = np.sort(np.concatenate([iu, ic, ip, im]))                     # a miss by (a) and a hit are done
    out = (depth, samples)
    if blocks:
        out += (np.concatenate(seen) if seen else np.zeros((0, 4), np.int64),)
    return out


def render(exp, voxel_size, vps, T, K, width, height, min_depth, max_depth, min_weight=1e-4):
    """-> dict with the keys and layout of Integrator.render(): depth [H, W], points_G [H, W, 3] and the point query at the hit"""
    depth, _ = march(exp, voxel_size, vps, T, K, width, height, min_depth, max_depth, min_weight)
    cam = Camera(T, K, width, height)
    hit = ~np.isnan(depth)
    pts = np.full((width * height, 3), qr.NAN_BITS, np.uint32).view(F)
    idx = np.nonzero(hit)[0]
    pts[idx] = cam.point(idx, depth[idx])
    out = {"depth": depth.reshape(height, width), "points_G": pts.reshape(height, width, 3)}
    q = qr.query(exp, voxel_size, vps, pts, min_weight)
    for k, v in q.items():
        out[k] = v.reshape((height, width) + v.shape[1:])
    return out
