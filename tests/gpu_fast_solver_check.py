"""Helper run in its own process by tests/test_gpu_fast_solver_edges.py, with KSG_SOLVE_THREADS set by the caller (it is read
when the integrator is created): the scenes of tests/fast_solver_scenes.py through the CUDA path and the oracle.

  parity:   every frame, bit-exact map, equal counters and equal updated() block sets; scenes 2-4 again after reset() and
            after clear_map().  REPORT {scene: [failures]}
  coverage: the same frames with profiling on.  REPORT {scene: [{sweeps, rays, rays_scanned, max_shared_slot_visitors}, ...]}"""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)


def scenes():
    import fast_solver_scenes as S
    from kimera_semantics_b200.capi import KSG_ORDER_SORTED
    # (name, (cfg, frames, None), whether the frames run again after reset() and clear_map())
    yield "aliased_start", S.scene_aliased_start(certificate=False), False
    yield "aliased_start_sorted", S.scene_aliased_start(order=KSG_ORDER_SORTED, certificate=False), False
    yield "overflow_fan", S.scene_overflow("fan", certificate=False), True
    yield "overflow_alias", S.scene_overflow("alias", certificate=False), True
    yield "window_edges_c0", S.scene_window_edges(0, certificate=False), True
    yield "window_edges_c2", S.scene_window_edges(2, certificate=False), True
    yield "deep_fixpoint", S.scene_deep_fixpoint(certificate=False), True


def parity_failures(gpu, ora, frame, where):
    """One frame through both integrators; the list of what differs (empty: counters, map bit for bit and updated() blocks equal).
    Also used by the in-process tests of test_gpu_fast_solver_edges.py, so both hold the same definition of parity."""
    import numpy as np
    from parity_utils import assert_parity, compare_maps, stats_equal
    T, xyz, labels, freespace = frame
    sg = gpu.integrate_points(T, xyz, labels=labels, freespace=freespace)
    so = ora.integrate_points(T, xyz, labels=labels, freespace=freespace)
    bad = []
    ok, why = stats_equal(sg, so)
    if not ok:
        bad.append(f"{where}: {why}")
    rep = compare_maps(gpu.export(), ora.export())
    try:
        assert_parity(rep, rtol=0.0)
    except AssertionError as e:
        bad.append(f"{where}: {str(e)[:300]}")
        return bad
    bits = {k: v for k, v in rep.items() if k.endswith("bit_mismatch") and v}
    if bits:
        bad.append(f"{where}: bit mismatches {bits}")
    if not np.array_equal(gpu.last_updated_blocks(), ora.last_updated_blocks()):
        bad.append(f"{where}: updated() block sets differ")
    return bad


def parity():
    from kimera_semantics_b200.capi import Integrator
    from oracle.oracle_py import OracleIntegrator
    report = {}
    for name, (cfg, frames, _), again in scenes():
        bad = []
        gpu, ora = Integrator(cfg), OracleIntegrator(cfg)
        try:
            for run in ("fresh", "after reset", "after clear_map") if again else ("fresh",):
                if run == "after reset":          # ksg_reset = a fresh integrator
                    gpu.reset()
                    ora.close()
                    ora = OracleIntegrator(cfg)
                elif run == "after clear_map":    # the approximate sets outlive the emptied map on both sides
                    gpu.clear_map()
                    ora.clear_map()
                for i, frame in enumerate(frames):
                    bad += parity_failures(gpu, ora, frame, f"{run} frame {i}")
        except Exception as e:   # a status code from the C-ABI
            bad.append(f"error: {str(e)[:300]}")
        gpu.close()
        ora.close()
        report[name] = bad
    return report


def coverage():
    from kimera_semantics_b200.capi import Integrator
    report = {}
    for name, (cfg, frames, _), _again in scenes():
        gpu = Integrator(cfg)
        gpu.set_profiling(True)
        out = []
        for T, xyz, labels, freespace in frames:
            gpu.integrate_points(T, xyz, labels=labels, freespace=freespace)
            tl = gpu.fast_timeline()
            d = tl["debug"]
            out.append({"sweeps": tl["sweeps"], "rays": d["rays"], "rays_scanned": d["rays_scanned"],
                        "max_shared_slot_visitors": d["max_shared_slot_visitors"]})
        gpu.close()
        report[name] = out
    return report


if __name__ == "__main__":
    mode = sys.argv[1]
    print("REPORT " + json.dumps(parity() if mode == "parity" else coverage()), flush=True)
