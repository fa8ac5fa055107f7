"""The certificates of tests/apply_edge_scenes.py, on the CPU: every scene reaches what it is named for (segment lengths exact to the
record, the routes, the weight and distance paths of tsdf_batch on hot, long and short segments), and the certificate describes the
scene the oracle sees: the oracle's voxel_updates equals the certificate's record total in every frame, and the camera voxel's
(distance, weight) in the oracle's map equals the state the branch model carried through the frames, bit for bit.  The scenes run on
the device in test_gpu_apply_edges.py."""
from collections import Counter

import numpy as np
import pytest

import apply_edge_scenes as S
from kimera_semantics_b200.capi import KSG_INTEGRATOR_FAST
from oracle.oracle_py import OracleIntegrator
from test_oracle_crosscheck import raycast


def oracle_frames(cfg, frames):
    ora = OracleIntegrator(cfg)
    stats = [ora.integrate_points(T, xyz, rgba=rgba, labels=labels, freespace=fs) for T, xyz, labels, fs, rgba in frames]
    exp = ora.export()
    ora.close()
    return stats, exp


def voxel_of_export(exp, vps, g):
    b = np.flatnonzero((exp["block_index"] == np.floor_divide(np.array(g), vps)).all(axis=1))[0]
    lx, ly, lz = (int(v) % vps for v in g)
    lin = lx + vps * (ly + vps * lz)
    return exp["tsdf_distance"][b, lin], exp["tsdf_weight"][b, lin]


def check_against_oracle(cfg, frames, cert):
    stats, exp = oracle_frames(cfg, frames)
    for st, c in zip(stats, cert):
        assert (st.rays_cast, st.voxel_updates) == (c["bundles"], c["records"])
    d, w = voxel_of_export(exp, cfg.voxels_per_side, cert[-1]["camera_voxel"])
    cd, cw, _ = cert[-1]["camera_voxel_state"]
    assert (d.tobytes(), w.tobytes()) == (np.float32(cd).tobytes(), np.float32(cw).tobytes()), (d, w, cd, cw)


def total_paths(cert):
    out = Counter()
    for c in cert:
        out.update(c["paths"])
    return out


def test_vectorised_raycaster_equals_the_serial_restatement():
    cfg, frames, _ = S.scene_route_edge(257, 21, certificate=False)
    T, xyz, _, _, _ = frames[0]
    origin = T[4:].astype(np.float32)
    for clearing in (False, True):
        pG, _, _ = S.bundles_of_frame(cfg, T, (xyz * np.float32(2.0 if clearing else 1.0)).astype(np.float32), clearing)
        ids, vox = S.raycast_many(cfg, origin, pG, np.full(len(pG), clearing))
        for b in range(0, len(pG), 16):
            want = raycast(origin, pG[b], clearing, np.float32(cfg.max_ray_length_m), np.float32(1.0 / np.float32(cfg.voxel_size)),
                           np.float32(cfg.default_truncation_distance), True)
            assert [tuple(v) for v in vox[ids == b]] == want, (clearing, b)


@pytest.mark.parametrize("C,n", [(C, n) for C, ns in S.ROUTE_EDGES.items() for n in ns])
def test_route_edges_are_exact(C, n):
    cfg, frames, cert = S.scene_route_edge(n, C)
    c = cert[0]
    llen = S.long_len(C)
    assert c["bundles"] == n and c["camera_voxel_records"] == n == max(c["lengths"])
    want = "hot" if n >= S.HOT_LEN else "long" if n >= llen else "short"
    assert c["routes"][want] >= 1 and (want == "hot") == (c["routes"]["hot"] == 1)
    if n < llen:
        assert c["routes"]["long"] == 0
    print(f"C={C} N={n}: route {want}, routes {c['routes']}, last batch {n % 32 or 32}, batches mod 3 = {-(-n // 32) % 3}, paths {c['paths']}")
    check_against_oracle(cfg, frames, cert)


def test_hot_route_edges_cover_the_pipeline_tails():
    ns = [n for n in S.ROUTE_EDGES[21] if n >= S.HOT_LEN]
    assert {-(-n // 32) % 3 for n in ns} == {0, 1, 2}            # the deep pipelines are unrolled by three batches
    assert {n % 32 or 32 for n in ns} >= {1, 32} and {n % 32 or 32 for n in S.ROUTE_EDGES[21]} >= {1, 31, 32}   # last batch


@pytest.mark.parametrize("variant", list(S.WEIGHT_VARIANTS))
def test_weight_states_cross_the_clamp_then_start_saturated(variant):
    cfg, frames, cert = S.scene_weight_states(variant)
    p0, p1 = Counter(cert[0]["paths"]), Counter(cert[1]["paths"])
    print(variant, "max_weight", cfg.max_weight, [c["paths"] for c in cert])
    assert all(c["camera_voxel_records"] == 4200 and c["routes"]["hot"] == 1 for c in cert)
    # frame 0: from weight 0 through the bare chain, across the clamp inside a batch, then saturated
    assert (variant == "low_max_weight" or p0["hot/wide/commit"] > 10) and p0["hot/saturated/commit"] > 10
    assert p0["hot/general/commit"] + p0["hot/general/replay"] >= 2
    if variant == "low_max_weight":
        assert p0["short/general/commit"] > 0 and p1["short/saturated/commit"] > 100
    # frames 1, 2: the whole hot segment starts saturated and pinned: the state hot_voxel_mode 2 skips
    for c in cert[1:]:
        assert c["paths"]["hot/saturated/commit"] == -(-4200 // 32) and sum(v for k, v in c["paths"].items() if k.startswith("hot/")) == -(-4200 // 32)
    assert cert[0]["camera_voxel_state"][:2] == (np.float32(cfg.default_truncation_distance), np.float32(cfg.max_weight))
    # with drop-off the last voxels of a ray get weight 0 (or below 1e-6) on a voxel of weight 0: the `new weight < 1e-6` skip
    assert (cert[0]["zero_weight_tail_records"] == 0) if variant == "no_dropoff" else (cert[0]["zero_weight_tail_records"] > 1000)
    assert sum(v for k, v in p1.items() if k.startswith("long/")) > 100
    check_against_oracle(cfg, frames, cert)


@pytest.mark.parametrize("variant", list(S.MOVING_VARIANTS))
def test_moving_distance_replays_long_segments(variant):
    cfg, frames, cert = S.scene_moving_distance(variant)
    print("moving distance", variant, [c["paths"] for c in cert])
    for c in cert[:2]:                                            # every batch of the hot and the long segments is replayed
        assert all(k.endswith("/replay") for k in c["paths"]), c["paths"]
        assert sum(v for k, v in c["paths"].items() if k.startswith("hot/")) == -(-4097 // 32)
    p = total_paths(cert)
    for route, bare in (("hot", "wide"), ("long", "unrolled"), ("short", "unrolled")):
        assert (p[f"{route}/{bare}/replay"] > 0 or variant == "color_low_max_weight") and p[f"{route}/general/replay"] > 0, route
    if variant == "semantic":
        assert p["hot/saturated/replay"] > 0 and p["hot/saturated/commit"] > 0 and p["long/saturated/replay"] > 0
    elif variant == "color":
        assert p["hot/partial/replay"] == 2 and p["hot/saturated/replay"] == 0
    else:
        assert p["short/saturated/replay"] > 0 and p["short/saturated/commit"] > 0
    assert cert[-1]["bundles"] > 4000 and cert[-1]["routes"]["hot"] == 1      # the freespace frame: clearing bundles
    check_against_oracle(cfg, frames, cert)


def test_scenes_together_reach_every_path_on_every_route():
    p = Counter()
    for name, build in S.all_scenes():
        if name.startswith(("route_edge_n4097_c21", "route_edge_n257_c21", "route_edge_n97_c33", "weight_states_default", "weight_states_low", "moving_distance_")):
            p.update(total_paths(build()[2]))
    print("paths over the scenes:", dict(sorted(p.items())))
    for route, bare in (("hot", "wide"), ("long", "unrolled"), ("short", "unrolled")):
        for w in (bare, "partial", "general", "saturated"):
            for d in S.M.DISTANCE_PATHS:
                assert p[f"{route}/{w}/{d}"] > 0, (route, w, d)


@pytest.mark.parametrize("C", S.CLASS_COUNTS)
def test_class_count_scenes(C):
    cfg, frames, cert = S.scene_class_count(C)
    assert cfg.num_labels == C and cert[0]["camera_voxel_records"] == 4097
    assert cert[0]["routes"]["hot"] == 1 and cert[0]["routes"]["long"] >= (10 if C <= 32 else 40)
    labels = np.concatenate([f[2] for f in frames])
    assert labels.min() == 0 and labels.max() == C - 1
    stats, _ = oracle_frames(cfg, frames)
    assert stats[0].voxel_updates == cert[0]["records"] and all(s.voxel_updates > 1000 for s in stats)


def test_fast_scene_saturates_and_blends():
    cfg, frames, _ = S.scene_fast_saturate()
    assert cfg.integrator_type == KSG_INTEGRATOR_FAST
    _, exp = oracle_frames(cfg, frames)
    w = exp["tsdf_weight"]
    assert (w == np.float32(cfg.max_weight)).sum() > 1000 and ((w > 0) & (w < np.float32(cfg.max_weight))).sum() > 1000
    assert (exp["tsdf_rgba"][w > 0][:, :3] != 0).any(axis=1).sum() > 1000
