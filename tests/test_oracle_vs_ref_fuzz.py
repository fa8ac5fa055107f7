"""Randomised differential test: the oracle against the reference's own sources (oracle/_ref) on random clouds, poses and
configuration switches - far/near/behind-the-camera points, |z| ~ 0 (zero weight), unknown colours, freespace clouds, every
Config flag.  Bit-exact in every exported field; `merged` in the oracle's faithful (libstdc++ bundle order) mode.  The reference's
maps are stored as digests (tests/golden/ref_extra_golden.json, tests/golden/make_ref_extra_golden.py); where oracle/_ref is
built, the live reference is compared as well.
The same generator (tests/fuzz_cases.py) drives the CUDA path in tests/test_gpu_fuzz.py."""
import importlib.util
import json
import os

import pytest

from oracle import ref_py
from oracle.oracle_py import OracleIntegrator
from parity_utils import compare_maps
import fuzz_cases

_spec = importlib.util.spec_from_file_location("make_ref_golden", os.path.join(os.path.dirname(__file__), "golden", "make_ref_golden.py"))
mrg = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(mrg)
GOLDEN = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "ref_extra_golden.json")))["fuzz"]


@pytest.mark.parametrize("seed", range(24))
def test_random_case_oracle_equals_reference_sources(seed):
    cfg, frames = fuzz_cases.make_case(seed)
    ora = OracleIntegrator(cfg, canonical_merged=False)
    ora.set_color_to_label(*fuzz_cases.color_table(cfg))
    ref = ref_py.RefHybridIntegrator(cfg) if ref_py.available() else None
    with fuzz_cases.quiet_stderr():
        for T, pts, rgba, freespace in frames:
            ora.integrate_points(T, pts, rgba=rgba, freespace=freespace)
            if ref is not None:
                ref.integrate_points(T, pts, rgba=rgba, freespace=freespace)
    got = mrg.digest(ora.export())
    for k in mrg.KEYS:
        assert got[k] == GOLDEN[str(seed)][k], f"seed {seed}: {k} differs from the reference's digest"
    assert got["order_insensitive"] == GOLDEN[str(seed)]["order_insensitive"]
    if ref is not None:
        rep = compare_maps(ref.export(), ora.export())
        assert rep["same_blocks"] == 1.0, rep
        assert not {k: v for k, v in rep.items() if k.endswith("mismatch") and v}, rep
