"""The device solver scans, after its first sweep, only a worklist: the rays evaluated in the previous sweep and the other rays
with an entry in a slot that sweep toggled (tools/observed_set_fixpoint.py: stamped_solve, DESIGN.md section 4).  Checked here
on real frame geometry against the sequential definition and against the scan of every ray in every sweep."""
import os
import sys

import numpy as np
import pytest

from kimera_semantics_b200 import synth
from kimera_semantics_b200.capi import KSG_INTEGRATOR_FAST
from parity_utils import frames, make_config
from test_fixpoint_prototype import cast_rays_of_frame
from test_oracle_crosscheck import ApproxSet

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))
import observed_set_fixpoint as fx  # noqa: E402


def table_after(rays, table, U):
    """Persistent table after the frame: every performed visit and breaking step writes its slot, in (rank, step) order."""
    t = dict(table)
    for vals, u in zip(rays, U):
        for s in fx.examined(vals, u):
            t[vals[s] & fx.MASK] = vals[s]
    return t


@pytest.mark.parametrize("max_collisions", [0, 2])
def test_worklist_sweeps_reach_the_sequential_result_and_scan_every_dirty_ray(max_collisions):
    C_, w, h = 5, 64, 48
    cfg = make_config(KSG_INTEGRATOR_FAST, 0.10, C_, max_points=w * h, max_consecutive_ray_collisions=max_collisions)
    start_set = ApproxSet()
    table = {0: (1 << 64) - 1}
    offset = 0
    rng = np.random.default_rng(5)
    for cam, depth, label, T in frames(w, h, C_, 3):
        offset += 1
        start_set.reset()
        xyz, pix = synth.backproject(depth, cam)
        rays = cast_rays_of_frame(cfg, T, xyz, label.reshape(-1)[pix], start_set, offset)
        assert len(rays) > 300
        U_seq, table_seq = fx.sequential(rays, table, max_collisions)
        lengths = [len(r) for r in rays]
        for U0 in ([min(L, max_collisions) for L in lengths], [int(rng.integers(0, L + 1)) for L in lengths]):
            U_w, n_w, log_w = fx.stamped_solve(rays, table, max_collisions, U0, worklist=True)
            U_f, n_f, log_f = fx.stamped_solve(rays, table, max_collisions, U0, worklist=False)
            assert U_w == U_seq and U_f == U_seq
            assert table_after(rays, table, U_w) == table_seq
            for scanned, evaluated, missing, stale in log_w + log_f:
                assert missing == [] and stale == []          # every dirty ray is listed; a clean ray would not change
            # the same evaluations as the full scan, sweep by sweep, from a far shorter scan
            assert n_w == n_f and [e for _, e, _, _ in log_w] == [e for _, e, _, _ in log_f]
            assert sum(s for s, _, _, _ in log_w) <= sum(s for s, _, _, _ in log_f)
            if n_w > 2:
                assert sum(s for s, _, _, _ in log_w[2:]) < sum(s for s, _, _, _ in log_f[2:])
        table = table_seq
