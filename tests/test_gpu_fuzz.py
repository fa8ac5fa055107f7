"""Randomised parity: the CUDA path through the C-ABI against the oracle on the seeded random clouds / poses / configurations of
tests/fuzz_cases.py (the oracle itself is held to the reference's own sources on the same cases in tests/test_oracle_vs_ref_fuzz.py).
Block set, labels, colours, distances, weights and log-probabilities must all be bit-exact, and the per-frame counters equal.

The cases cover saturating max_weight, odd voxel sizes, points behind the camera, zero-weight points, random orientations, ...;
they run in their own process, so a corner case that needs work has no effect on the rest of the suite."""
import json
import os
import subprocess
import sys

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.mark.gpu
def test_random_cases_cuda_path_equals_oracle_bit_for_bit():
    r = subprocess.run([sys.executable, os.path.join(HERE, "gpu_fuzz_check.py"), "0", "24"], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr[-2000:]
    line = [l for l in r.stdout.splitlines() if l.startswith("REPORT ")][-1]
    report = json.loads(line[len("REPORT "):])
    assert len(report) == 24
    bad = {s: e for s, e in report.items()
           if "error" in e or e.get("same_blocks") != 1.0 or not e.get("stats_ok") or any(v for k, v in e.items() if k.endswith("mismatch"))}
    assert not bad, bad
