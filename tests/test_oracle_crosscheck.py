"""A second, independent restatement (numpy float32, written from SURVEY.md Appendix A, sharing no code with
oracle/ks_oracle.cpp) of the pieces that decide WHICH voxels a frame touches: quaternion transform (A.8), grid index (A.2),
RayCaster (A.7), ThreadSafeIndex "mixed" (A.3), ApproxHashSet (A.4) and the fast integrator's control flow (fast.cpp:57-143).
It replays a small frame and must reproduce the oracle's per-frame counters and touched-voxel set exactly."""
import numpy as np
import pytest

from kimera_semantics_b200 import synth
from kimera_semantics_b200.capi import KSG_INTEGRATOR_FAST, KSG_INTEGRATOR_MERGED
from oracle.oracle_py import OracleIntegrator
from parity_utils import frames, make_config

f32 = np.float32
EPS = f32(1e-6)


def transform(T, p):
    qw, qx, qy, qz = (f32(v) for v in T[:4])
    t = T[4:].astype(np.float32)
    qv = np.array([qx, qy, qz], np.float32)

    def cross(a, b):
        return np.array([f32(f32(a[1] * b[2]) - f32(a[2] * b[1])), f32(f32(a[2] * b[0]) - f32(a[0] * b[2])), f32(f32(a[0] * b[1]) - f32(a[1] * b[0]))], np.float32)
    uv = cross(qv, p)
    uv = (uv + uv).astype(np.float32)
    r = ((p + (uv * qw).astype(np.float32)).astype(np.float32) + cross(qv, uv)).astype(np.float32)
    return (r + t).astype(np.float32)


def norm(v):
    return f32(np.sqrt(f32(f32(f32(v[0] * v[0]) + f32(v[1] * v[1])) + f32(v[2] * v[2]))))


def grid_index(p, inv):
    return tuple(int(np.floor(f32(f32(p[k] * inv) + EPS))) for k in range(3))


def raycast(origin, pG, clearing, max_len, vsi, trunc, from_origin):
    return list(walk(origin, pG, clearing, max_len, vsi, trunc, from_origin))


def walk(origin, pG, clearing, max_len, vsi, trunc, from_origin):
    """The voxels of raycast(), one at a time (a caller that breaks early skips the rest of the walk)."""
    d = (pG - origin).astype(np.float32)
    n = norm(d)
    unit = (d / n).astype(np.float32) if n > 0 else d
    if clearing:
        L = f32(min(max(f32(n - trunc), f32(0)), max_len))
        end = (origin + (unit * L).astype(np.float32)).astype(np.float32)
        start = origin
    else:
        end = (pG + (unit * trunc).astype(np.float32)).astype(np.float32)
        start = origin
    s, e = (start * vsi).astype(np.float32), (end * vsi).astype(np.float32)
    if not from_origin:
        s, e = e, s
    cur = [int(np.floor(f32(s[k] + EPS))) for k in range(3)]
    endi = [int(np.floor(f32(e[k] + EPS))) for k in range(3)]
    steps = sum(abs(endi[k] - cur[k]) for k in range(3))
    r = (e - s).astype(np.float32)
    sign = [int(r[k] > 0) - int(r[k] < 0) for k in range(3)]
    with np.errstate(divide="ignore", invalid="ignore"):
        tn = [f32(f32(f32(max(0, sign[k])) - f32(s[k] - f32(cur[k]))) / r[k]) for k in range(3)]
        ts = [f32(f32(sign[k]) / r[k]) for k in range(3)]
    for _ in range(steps + 1):
        yield tuple(cur)
        k = 0
        if tn[1] < tn[k]:
            k = 1
        if tn[2] < tn[k]:
            k = 2
        cur[k] += sign[k]
        tn[k] = f32(tn[k] + ts[k])


def index_hash(g):
    return (g[0] + g[1] * 17191 + g[2] * 17191 * 17191) % (1 << 64) % (1 << 32)


class ApproxSet:
    def __init__(self):
        self.table = {0: (1 << 64) - 1}
        self.offset = 0

    def replace(self, h):
        v = h + self.offset
        k = v & 0xFFFFF
        if self.table.get(k, 0) == v:
            return False
        self.table[k] = v
        return True

    def reset(self):
        self.offset += 1
        if self.offset >= 10000:
            self.__init__()


def mixed_order(n):
    groups = n // 1024
    return [s if groups * 1024 <= s else (s % groups) * 1024 + s // groups for s in range(n)]


def sorted_order(xyz):
    """SortedThreadSafeIndex (A.3): by squared range, ties by index."""
    x = np.asarray(xyz, np.float32)
    sq = ((x[:, 0] * x[:, 0] + x[:, 1] * x[:, 1]).astype(np.float32) + x[:, 2] * x[:, 2]).astype(np.float32)
    return np.argsort(sq, kind="stable").tolist()


class FastReplay:
    """fast.cpp:57-199 control flow only (which voxels get an update), no voxel arithmetic.  `touched` collects every frame's updated
    voxels, `frame_touched` those of the last frame."""

    def __init__(self, cfg):
        self.cfg = cfg
        self.start, self.obs = ApproxSet(), ApproxSet()
        self.vsi = f32(1.0 / f32(cfg.voxel_size))
        self.touched = set()
        self.frame_touched = set()
        self.reset_counter = 0

    def integrate(self, T, xyz, labels, freespace=False):
        c = self.cfg
        self.reset_counter += 1
        if self.reset_counter >= c.clear_checks_every_n_frames:     # fast.cpp:165-171
            self.reset_counter = 0
            self.start.reset(); self.obs.reset()
        self.frame_touched = set()
        allow_clear = c.allow_clear and c.voxel_carving_enabled
        origin = T[4:].astype(np.float32)
        updates = rays = valid = 0
        start_inv = f32(f32(c.start_voxel_subsampling_factor) * self.vsi)
        order = sorted_order(xyz) if c.integration_order_mode == 1 else mixed_order(len(xyz))
        for i in order:
            p = xyz[i]
            rng = norm(p)
            if rng < f32(c.min_ray_length_m):
                continue
            clearing = bool(freespace)
            if rng > f32(c.max_ray_length_m):
                if not (allow_clear or freespace):
                    continue
                clearing = True
            if c.dynamic_label[int(labels[i])]:
                continue
            valid += 1
            pG = transform(T, p)
            if not self.start.replace(index_hash(grid_index(pG, start_inv))):
                continue
            rays += 1
            run = 0
            for g in walk(origin, pG, clearing, f32(c.max_ray_length_m), self.vsi, f32(c.default_truncation_distance), False):
                if not self.obs.replace(index_hash(g)):
                    run += 1
                else:
                    run = 0
                if run > c.max_consecutive_ray_collisions:
                    break
                self.touched.add(g)
                self.frame_touched.add(g)
                updates += 1
        return valid, rays, updates


def touched_voxels(exp, vps):
    out = set()
    upd = np.argwhere((exp["sem_priors"] < np.float32(-0.60205999132)).any(axis=-1) | (exp["tsdf_weight"] > 0))
    for b, lin in upd:
        bx, by, bz = (int(v) for v in exp["block_index"][b])
        out.add((bx * vps + lin % vps, by * vps + (lin // vps) % vps, bz * vps + lin // (vps * vps)))
    return out


def test_fast_control_flow_replay_matches_oracle_counters_and_touched_voxels():
    C_, w, h = 5, 96, 72
    cfg = make_config(KSG_INTEGRATOR_FAST, 0.10, C_, max_points=w * h)
    ora, rep = OracleIntegrator(cfg), FastReplay(cfg)
    for cam, depth, label, T in frames(w, h, C_, 3):
        xyz, pix = synth.backproject(depth, cam)
        lab = label.reshape(-1)[pix]
        so = ora.integrate_points(T, xyz, labels=lab)
        valid, rays, updates = rep.integrate(T, xyz, lab)
        assert (valid, rays, updates) == (so.points_valid, so.rays_cast, so.voxel_updates)
    # every voxel the replay updated carries an observation in the oracle's map. (Voxels that only ever saw label 0 with
    # zero TSDF weight are invisible in an export, hence subset + a tight size bound instead of equality.)
    tv = touched_voxels(ora.export(), 16)
    assert tv <= rep.touched and len(rep.touched) - len(tv) <= 0.02 * len(rep.touched) + 5


def test_merged_bundle_count_matches_independent_voxel_bucketing():
    """bundleRays (A.5): number of bundles = number of distinct (clearing, voxel) buckets of the valid points."""
    C_, w, h = 5, 96, 72
    cfg = make_config(KSG_INTEGRATOR_MERGED, 0.10, C_, max_points=w * h)
    ora = OracleIntegrator(cfg)
    vsi = f32(1.0 / f32(cfg.voxel_size))
    for cam, depth, label, T in frames(w, h, C_, 2):
        xyz, pix = synth.backproject(depth, cam)
        st = ora.integrate_points(T, xyz, labels=label.reshape(-1)[pix])
        buckets = set()
        for p in xyz:
            rng = norm(p)
            if rng < f32(cfg.min_ray_length_m):
                continue
            buckets.add((bool(rng > f32(cfg.max_ray_length_m)), grid_index(transform(T, p), vsi)))
        assert st.rays_cast == len(buckets)
