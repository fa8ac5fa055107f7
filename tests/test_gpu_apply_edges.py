"""The voxel-update kernels (ksg_voxel.cuh, tsdf_batch, k_tile_apply, k_tile_apply_fast) on the scenes of tests/apply_edge_scenes.py,
which put real voxels into the states where those kernels switch paths: segment lengths at the short / long / hot thresholds, weights
that start at zero, cross the clamp inside a batch and start saturated, distances that move on every record of a hot segment, class
counts at the kernel switches.  tests/test_apply_edge_scenes_cpu.py proves on the CPU which paths each scene takes.

Every frame of every scene is compared with the oracle bit for bit (counters, every exported field, updated() blocks), under the
default routes and again under each in-tree alternative: KSG_MERGED_TILE_APPLY=1, KSG_LONG_LEN=4096 (each set only around the
creation of the one integrator it is for, in a helper process that starts without them), apply_mode 1, hot_voxel_mode 1 and 2 and
the reference's bundle order.  The voxels the device queued per route (ksg_debug_apply_routes) must equal the certificate's counts,
and hot_voxel_mode 2 must actually skip the saturated camera voxel."""
import json
import os
import subprocess
import sys

import pytest

import apply_edge_scenes as S
from gpu_apply_edge_check import CFG_VARIANTS, ENV_VARIANTS, SUBSET

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope="module")
def report():
    env = {k: v for k, v in os.environ.items() if k not in ENV_VARIANTS}
    r = subprocess.run([sys.executable, os.path.join(HERE, "gpu_apply_edge_check.py")], capture_output=True, text=True, timeout=900,
                       env=env)
    assert r.returncode == 0, r.stderr[-2000:]
    line = [l for l in r.stdout.splitlines() if l.startswith("REPORT ")][-1]
    return json.loads(line[len("REPORT "):])


def check(report, names):
    assert set(names) <= set(report), sorted(set(names) - set(report))
    bad = {k: report[k]["failures"] for k in names if report[k]["failures"]}
    assert not bad, bad
    for name in names:
        r = report[name]
        if "expected_routes" in r:
            got = [{k: f[k] for k in ("hot", "long", "short")} for f in r["routes"][:len(r["expected_routes"])]]
            assert got == r["expected_routes"], name
    print(f"{len(names)} scene x configuration runs bit exact, e.g. {names[0]}: frame 0 routed {report[names[0]]['routes'][:1]}")


def test_every_scene_is_bit_exact_and_routed_as_certified(report):
    names = [n for n, _ in S.all_scenes()]
    check(report, names)
    assert (report["route_edge_n4096_c21"]["routes"][0]["hot"], report["route_edge_n4095_c21"]["routes"][0]["hot"]) == (1, 0)
    assert (report["route_edge_n256_c21"]["routes"][0]["long"], report["route_edge_n255_c21"]["routes"][0]["long"]) == (1, 0)
    assert (report["route_edge_n96_c33"]["routes"][0]["long"], report["route_edge_n95_c33"]["routes"][0]["long"]) == (1, 0)


@pytest.mark.parametrize("variant", list(CFG_VARIANTS))
def test_configuration_variants_are_bit_exact_and_routed_as_certified(report, variant):
    check(report, [f"{n}/{variant}" for n in SUBSET if not (variant.startswith("hot_voxel") and n.endswith("_c33"))])


def test_hot_voxel_mode_2_skips_the_saturated_camera_voxel_and_only_that(report):
    for name in ("weight_states_default", "weight_states_low_max_weight"):
        assert report[f"{name}/hot_voxel_mode_1"]["hot_voxels"] == [1, 1, 1], name
        r = report[f"{name}/hot_voxel_mode_2"]
        # frame 0 starts the camera voxel at weight 0; frames 1 and 2 start it at (+truncation, max_weight): the skip is taken
        assert [f["hot_tsdf_skipped"] for f in r["routes"]] == [0, 1, 1], (name, r["routes"])
    r = report["moving_distance_semantic/hot_voxel_mode_2"]       # saturated, but the distance moves: the skip must be refused
    assert [f["hot_tsdf_skipped"] for f in r["routes"]][:3] == [0, 0, 0], r["routes"]


@pytest.mark.parametrize("var", list(ENV_VARIANTS))
def test_alternative_routes_are_bit_exact_and_routed_as_certified(report, var):
    check(report, [f"{n}/{var}={ENV_VARIANTS[var]}" for n in SUBSET])
