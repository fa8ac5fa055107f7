"""`merged` in the reference's bundle order (ksg_config.merged_bundle_order = KSG_BUNDLE_ORDER_LIBSTDCXX): every exported field
must hash to the digest of the reference's own sources - the one place where the default product deviates from the
single-threaded reference (canonical first-insertion order, DESIGN.md section 4).

The order algorithm is proven on the CPU against the real container in tests/test_unordered_map_order.py.  The check runs in a
subprocess (the mode is young: a device fault would stay contained instead of poisoning the CUDA context of the suite)."""
import json
import os
import subprocess
import sys

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.mark.gpu
def test_merged_in_libstdcxx_bundle_order_equals_the_reference_sources_bit_for_bit():
    r = subprocess.run([sys.executable, os.path.join(HERE, "gpu_bundle_order_check.py")], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr[-2000:]
    line = [l for l in r.stdout.splitlines() if l.startswith("REPORT ")][-1]
    report = json.loads(line[len("REPORT "):])
    assert len(report) >= 10
    bad = {n: [k for k, ok in f.items() if not ok] for n, f in report.items() if not all(f.values())}
    assert not bad, bad
