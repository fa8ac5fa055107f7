"""Helper run in its own process by tests/test_gpu_merged_update_log.py: the update log of the `merged` integrator on the scenes of
tests/apply_edge_scenes.py (hot voxels of 4096+ records, segments on the 96 / 256 thresholds) under every apply route.  The KSG_* route
variables are read when an integrator is created, so each is set around that one creation and removed again; the process starts
without any of them.

REPORT {scene: {configuration: [per frame: [entries, sha256 of the entries, sha256 of the log-probability rows, sha256 of the exported
map, whether every entry equals the exported voxel]]}}; the configuration "default_again" is a second integrator under the default
routes.  Frame 0 of every scene under the default routes is also checked against the traced voxels (merged_update_trace.py):
"failures"."""
import hashlib
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

SCENES = ("route_edge_n255_c21", "route_edge_n256_c21", "route_edge_n4095_c21", "route_edge_n4096_c21", "route_edge_n4160_c21",
          "route_edge_n96_c33", "weight_states_default", "moving_distance_semantic", "class_count_merged_c33")
CFG_VARIANTS = {"apply_mode_1": {"apply_mode": 1}, "hot_voxel_mode_1": {"hot_voxel_mode": 1}, "hot_voxel_mode_2": {"hot_voxel_mode": 2}}
ENV_VARIANTS = {"KSG_MERGED_TILE_APPLY": 1, "KSG_LONG_LEN": 4096}


def values_match(heads, pri, exp):
    """Every entry's state equals the exported voxel, bit for bit."""
    import numpy as np
    row = {tuple(b): i for i, b in enumerate(exp["block_index"].tolist())}
    b = np.array([row[tuple(x)] for x in heads["block_index"].tolist()], np.int64)
    lin = (heads["lin_label"] & 0xFFFFFF).astype(np.int64)
    return bool(np.array_equal(heads["tsdf_distance"].view(np.uint32), exp["tsdf_distance"][b, lin].view(np.uint32))
                and np.array_equal(heads["tsdf_weight"].view(np.uint32), exp["tsdf_weight"][b, lin].view(np.uint32))
                and np.array_equal(heads["tsdf_rgba"], exp["tsdf_rgba"][b, lin]) and np.array_equal(heads["sem_rgba"], exp["sem_rgba"][b, lin])
                and np.array_equal(heads["lin_label"] >> 24, exp["sem_label"][b, lin])
                and np.array_equal(pri.view(np.uint32), exp["sem_priors"][b, lin].view(np.uint32)))


def run(cfg, frames, env, check=None):
    from kimera_semantics_b200.capi import Integrator
    os.environ.update({k: str(v) for k, v in env.items()})
    try:
        gpu = Integrator(cfg)
    finally:
        for k in env:
            del os.environ[k]
    gpu.set_update_log(1 << 20)
    out = []
    for i, (T, xyz, labels, freespace, rgba) in enumerate(frames):
        gpu.integrate_points(T, xyz, rgba=rgba, labels=labels, freespace=freespace)
        heads, pri = gpu.fetch_update_log()
        exp = gpu.export()
        mh = hashlib.sha256(b"".join(exp[k].tobytes() for k in sorted(exp))).hexdigest()
        out.append([len(heads), hashlib.sha256(heads.tobytes()).hexdigest(), hashlib.sha256(pri.tobytes()).hexdigest(), mh,
                    values_match(heads, pri, exp)])
        if check is not None and i == 0:
            check(gpu, frames[0], heads, pri)
    gpu.close()
    return out


def main():
    import apply_edge_scenes as S
    import merged_update_trace as tr
    assert not any(k in os.environ for k in ENV_VARIANTS), "route variables set in the caller's environment"
    builders = dict(S.all_scenes(certificate=False))
    report = {}
    for name in SCENES:
        cfg, frames, _ = builders[name](certificate=False)
        failures = []

        def check(gpu, frame, heads, pri):
            T, xyz, labels, freespace, rgba = frame
            want = tr.pairs(*tr.updated_voxels_points(cfg, T, xyz, freespace=freespace))
            got = tr.pairs(heads["block_index"], heads["lin_label"] & 0xFFFFFF)
            if len(got) != len(heads) or got != want:
                failures.append(f"log voxels: {len(heads)} entries, {len(got)} distinct, {len(want)} traced, {len(got ^ want)} differ")

        r = {"default": run(cfg, frames, {}, check), "default_again": run(cfg, frames, {})}
        for k, v in CFG_VARIANTS.items():
            if k.startswith("hot_voxel") and cfg.num_labels > 32:
                continue
            for a, x in v.items():
                setattr(cfg, a, x)
            r[k] = run(cfg, frames, {})
            for a in v:
                setattr(cfg, a, 0)
        for k, v in ENV_VARIANTS.items():
            r[f"{k}={v}"] = run(cfg, frames, {k: v})
        report[name] = {"runs": r, "failures": failures}
        print(f"{name}: {len(r)} configurations", file=sys.stderr, flush=True)
    return report


if __name__ == "__main__":
    print("REPORT " + json.dumps(main()), flush=True)
