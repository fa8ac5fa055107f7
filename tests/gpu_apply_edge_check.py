"""Helper run in its own process by tests/test_gpu_apply_edges.py: the scenes of tests/apply_edge_scenes.py through the CUDA path and
the oracle.  Every scene runs under the default routes; the scenes of SUBSET run again with apply_mode 1, hot_voxel_mode 1 and 2 and
the reference's bundle order, and under each KSG_* route variable of ENV_VARIANTS.  Those variables are read when an integrator is
created, so each is set around that one creation and removed again; the process starts without any of them.  The oracle integrates a
scene once per bundle order and its per-frame results are reused for every configuration.

REPORT {scene[/configuration]: {"failures": [...], "routes": [per frame], "expected_routes": [per certified frame], "hot_voxels": [...]}}
Every frame: counters, the whole exported map bit for bit, and the updated() block sets equal to the oracle's."""
import json
import os
import sys
import time

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

SUBSET = ("route_edge_n256_c21", "route_edge_n4095_c21", "route_edge_n4096_c21", "route_edge_n4097_c21", "route_edge_n4160_c21",
          "route_edge_n96_c33", "weight_states_default", "weight_states_low_max_weight", "moving_distance_semantic",
          "class_count_merged_c33")
CFG_VARIANTS = {"apply_mode_1": {"apply_mode": 1}, "hot_voxel_mode_1": {"hot_voxel_mode": 1}, "hot_voxel_mode_2": {"hot_voxel_mode": 2},
                "libstdcxx_bundle_order": {"merged_bundle_order": 1}}
ENV_VARIANTS = {"KSG_MERGED_TILE_APPLY": 1, "KSG_LONG_LEN": 4096}


def oracle_frames(cfg, frames):
    """Per frame: (stats, exported map, updated() blocks) of the oracle."""
    from oracle.oracle_py import OracleIntegrator
    ora = OracleIntegrator(cfg)
    out = []
    for T, xyz, labels, freespace, rgba in frames:
        so = ora.integrate_points(T, xyz, rgba=rgba, labels=labels, freespace=freespace)
        out.append((so, ora.export(), ora.last_updated_blocks()))
    ora.close()
    return out


def frame_failures(gpu, want, frame, where):
    import numpy as np
    from parity_utils import assert_parity, compare_maps, stats_equal
    T, xyz, labels, freespace, rgba = frame
    so, exp, updated = want
    sg = gpu.integrate_points(T, xyz, rgba=rgba, labels=labels, freespace=freespace)
    bad = []
    ok, why = stats_equal(sg, so)
    if not ok:
        bad.append(f"{where}: {why}")
    got = gpu.export()
    if all(got[k].shape == exp[k].shape and np.array_equal(got[k].view(np.uint8), exp[k].view(np.uint8)) for k in exp):
        rep = None                            # every exported field equal byte for byte
    else:
        rep = compare_maps(got, exp)
    if not np.array_equal(gpu.last_updated_blocks(), updated):
        bad.append(f"{where}: updated() block sets differ")
    if rep is None:
        return sg, bad
    try:
        assert_parity(rep, rtol=0.0)
    except AssertionError as e:
        return sg, bad + [f"{where}: {str(e)[:300]}"]
    bits = {k: v for k, v in rep.items() if k.endswith("bit_mismatch") and v}
    bad.append(f"{where}: bit mismatches {bits}")
    return sg, bad


def run_scene(cfg, frames, want, env):
    from kimera_semantics_b200.capi import KSG_INTEGRATOR_MERGED, Integrator
    out = {"failures": [], "routes": [], "hot_voxels": []}
    gpu = None
    try:
        os.environ.update({k: str(v) for k, v in env.items()})
        try:
            gpu = Integrator(cfg)
        finally:
            for k in env:
                del os.environ[k]
        for i, frame in enumerate(frames):
            sg, bad = frame_failures(gpu, want[i], frame, f"frame {i}")
            out["failures"] += bad
            out["hot_voxels"].append(int(sg.hot_voxels))
            if cfg.integrator_type == KSG_INTEGRATOR_MERGED:
                out["routes"].append(gpu.apply_routes())
    except Exception as e:   # a status code from the C-ABI
        out["failures"].append(f"error: {str(e)[:300]}")
    if gpu is not None:
        gpu.close()
    return out


def expected_routes(cfg, cert, env):
    """The certificate's route counts under the routes the configuration selects."""
    import apply_edge_scenes as S
    if cfg.apply_mode == 1 or int(env.get("KSG_MERGED_TILE_APPLY", 0)) != 0:
        return [{"hot": 0, "long": 0, "short": 0} for _ in cert]            # the tile kernel: no queues
    llen = S.long_len(cfg.num_labels, env_long_len=env.get("KSG_LONG_LEN"))
    return [S.routes(c["lengths"], llen) for c in cert]


def main():
    import apply_edge_scenes as S
    assert not any(k in os.environ for k in ENV_VARIANTS), "route variables set in the caller's environment"
    report = {}
    for name, build in S.all_scenes():
        t0 = time.time()
        cfg, frames, cert = build(certificate=True)
        configs = [("", {}, {})]
        if name in SUBSET:
            configs += [("/" + k, v, {}) for k, v in CFG_VARIANTS.items() if not (k.startswith("hot_voxel") and cfg.num_labels > 32)]
            configs += [(f"/{k}={v}", {}, {k: v}) for k, v in ENV_VARIANTS.items()]
        want = {}
        for tag, kw, env in configs:
            for k, v in kw.items():
                setattr(cfg, k, v)
            if cfg.merged_bundle_order not in want:
                want[cfg.merged_bundle_order] = oracle_frames(cfg, frames)
            r = run_scene(cfg, frames, want[cfg.merged_bundle_order], env)
            if cert is not None:
                r["expected_routes"] = expected_routes(cfg, cert, env)
            for k in kw:
                setattr(cfg, k, 0)
            report[name + tag] = r
        print(f"{name}: {time.time() - t0:.1f} s, {len(configs)} configurations", file=sys.stderr, flush=True)
    return report


if __name__ == "__main__":
    print("REPORT " + json.dumps(main()), flush=True)
