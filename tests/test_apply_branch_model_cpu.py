"""tests/apply_branch_model.py on the CPU: the numpy restatement of tsdf_batch equals the sequential definition on every family (this
extends test_weight_chain_bound.py from the weight chain to the distance speculation and the colour), and the families together
take every (weight path, distance path) of the kernel, and each family the path its name says.  The same families run through the
kernel in test_gpu_tsdf_batch.py."""
from collections import Counter

import numpy as np
import pytest

import apply_branch_model as M

FAMILIES = M.families()


def paths_of(name, wide=False):
    f = next(f for f in FAMILIES if f["name"] == name)
    return M.run_family(f, wide)[3:]


def test_model_equals_the_sequential_definition_on_every_family():
    assert len({f["name"] for f in FAMILIES}) == len(FAMILIES)
    for f in FAMILIES:
        ref = M.run_sequential(f)
        for wide in (False, True):
            got = M.run_family(f, wide)
            assert M.same_state(got, ref), (f["name"], wide, got[:3], ref)


def test_families_take_every_weight_and_distance_path():
    total = {False: Counter(), True: Counter()}
    for f in FAMILIES:
        for wide in (False, True):
            total[wide] += M.run_family(f, wide)[3]
    for wide in (False, True):
        print(f"wide={int(wide)}:", {f"{w}/{d}": total[wide][(w, d)] for w in M.WEIGHT_PATHS for d in M.DISTANCE_PATHS})
    for d in M.DISTANCE_PATHS:
        for w in ("saturated", "partial", "general"):
            assert total[False][(w, d)] > 0 and total[True][(w, d)] > 0, (w, d)
        assert total[False][("unrolled", d)] > 0 and total[True][("wide", d)] > 0, d
        assert total[False][("wide", d)] == 0 and total[True][("unrolled", d)] == 0


def test_lengths_and_max_weights_are_all_present():
    for n in M.LENGTHS:
        assert any(len(f["sdf"]) == n for f in FAMILIES), n
    for mw in M.MAX_WEIGHTS:
        assert any(f["max_weight"] == M.F(mw) for f in FAMILIES), mw
    long_chain = sum((M.run_family(f, True)[3] for f in FAMILIES if len(f["sdf"]) >= 4096), Counter())
    for w in ("saturated", "wide", "general"):                  # a chain of hot-voxel length crosses the clamp on its way
        assert sum(long_chain[(w, d)] for d in M.DISTANCE_PATHS) > 0, w
    assert long_chain[("wide", "replay")] > 32 and long_chain[("wide", "commit")] > 32


@pytest.mark.parametrize("max_w", M.MAX_WEIGHTS)
def test_named_weight_paths(max_w):
    for kind in ("pinned", "moving"):
        p, _ = paths_of(f"saturated_{kind}_max{max_w:g}")
        assert {w for w, _ in p} == {"saturated"} and sum(p.values()) == 3
    f = next(f for f in FAMILIES if f["name"] == f"saturated_one_negative_max{max_w:g}")
    first = M.run_family(dict(f, sdf=f["sdf"][:32], uw=f["uw"][:32]), False)[3]
    both = M.run_family(dict(f, sdf=f["sdf"][:64], uw=f["uw"][:64]), False)[3]
    assert {w for w, _ in first} == {"saturated"} and {w for w, _ in both - first} == {"general"}     # the skip is refused once
    for nb, bare in ((32, "unrolled"), (20, "partial")):
        assert {w for w, _ in paths_of(f"margin_below_nb{nb}_max{max_w:g}")[0]} == {bare}
        assert {w for w, _ in paths_of(f"margin_above_nb{nb}_max{max_w:g}")[0]} == {"general"}
        f_lo = next(f for f in FAMILIES if f["name"] == f"margin_below_nb{nb}_max{max_w:g}")
        f_hi = next(f for f in FAMILIES if f["name"] == f"margin_above_nb{nb}_max{max_w:g}")
        ulps = np.abs(f_lo["uw"].view(np.int32).astype(np.int64) - f_hi["uw"].view(np.int32)).max()
        assert ulps <= 2, ulps                                   # the two sides of the bound are a few ulp apart
    assert {w for w, _ in paths_of(f"margin_below_nb32_max{max_w:g}", wide=True)[0]} == {"wide"}
    for k in (0, 15, 31):
        f = next(f for f in FAMILIES if f["name"] == f"clamp_at_record{k}_max{max_w:g}")
        p, _ = M.run_family(f, False)[3:]
        assert sum(c for (w, _), c in p.items() if w == "unrolled") == 1 and sum(c for (w, _), c in p.items() if w == "general") == 1
        assert sum(c for (w, _), c in p.items() if w == "saturated") == 1
        # the weight is below the clamp before record k of the second batch and at it afterwards
        before = M.sequential(f["trunc"], f["max_weight"], f["sdf"][:32 + k], f["uw"][:32 + k], None, False, f["dist"], f["wgt"], 0)[1]
        after = M.sequential(f["trunc"], f["max_weight"], f["sdf"][:33 + k], f["uw"][:33 + k], None, False, f["dist"], f["wgt"], 0)[1]
        assert before < f["max_weight"] == after
    p, _ = paths_of(f"clamp_in_last_batch_max{max_w:g}")
    assert p == Counter({("unrolled", "commit"): 1, ("general", "commit"): 1})


def test_named_distance_paths():
    for name in ("pinned_plus", "pinned_minus"):
        p, movers = paths_of(name)
        assert {d for _, d in p} == {"commit"} and not movers, name
    for k in (0, 1, 31, 67):
        p, movers = paths_of(f"first_mover_at_record{k}")
        assert movers[0] == (k // 32, k % 32), (k, movers)      # every batch before the mover's commits whole
    p, movers = paths_of("every_record_moves")
    assert {d for _, d in p} == {"replay"} and all(m[1] == 0 for m in movers)
    f = next(f for f in FAMILIES if f["name"] == "cancel_to_plus_zero")
    d = M.sequential(f["trunc"], f["max_weight"], f["sdf"][:1], f["uw"][:1], None, False, f["dist"], f["wgt"], 0)[0]
    assert np.array(d, M.F).tobytes() == M.F(0.0).tobytes()
    p, movers = paths_of("cancel_from_minus_zero")
    assert movers and movers[0] == (0, 0)                        # -0 -> +0 is a change of bits: the record counts as a mover


def test_start_weights_around_the_skip_threshold():
    for tag in ("zero", "below_eps", "eps", "above_eps"):
        f = next(f for f in FAMILIES if f["name"] == f"start_{tag}_tiny_weights")
        skipped = 0
        w = f["wgt"]
        for u in f["uw"]:
            nw = M.F(w + u)
            if nw < M.EPS:
                skipped += 1
            else:
                w = min(f["max_weight"], nw)
        assert (skipped > 0) == (tag in ("zero", "below_eps")), (tag, skipped)
        for kind in ("one_nan", "one_negative"):
            p, _ = paths_of(f"start_{tag}_{kind}")
            assert sum(c for (w_, _), c in p.items() if w_ == "general") >= 1


def test_blend_families_blend_only_near_the_surface():
    for f in FAMILIES:
        if not f["blend"]:
            continue
        ref = M.run_sequential(f)
        assert ref[2] != f["rgba"], f["name"]
        far_only = dict(f, sdf=np.where(np.abs(f["sdf"]) < f["trunc"], M.F(1.0), f["sdf"]))
        assert M.run_sequential(far_only)[2] == f["rgba"], f["name"]
