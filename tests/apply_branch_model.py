"""The TSDF recurrence of the warp-level apply kernels (tsdf_batch, csrc/ksg_kernels.cuh) restated in numpy float32, branch by branch,
next to the sequential definition it must equal (tsdf_chain_step, csrc/ksg_device.cuh = voxblox updateTsdfVoxel, SURVEY.md A.6).

tsdf_batch takes one of five ways through the weight chain of a batch of <= 32 records,

  saturated   the voxel sits at max_weight and no weight of the batch is negative or NaN: the chain is skipped
  wide        bare chain of additions, all 32 weights in registers first (the deep-pipeline instance, full batch)
  unrolled    bare chain, unrolled (full batch)
  partial     bare chain, partial batch
  general     the chain with the `new weight < 1e-6` skip and the clamp to max_weight

and one of two through the distance,

  commit      no record moves the clamped distance: the whole batch commits speculatively
  replay      the first record that moves it ends the speculation; the records behind it are replayed in order

`batch_walk` returns the final state and how many batches took each (weight path, distance path); `sequential` is the definition.
`families()` are seeded record chains, each built for the path its name says; tests/test_apply_branch_model_cpu.py proves on the CPU
that they reach every path and that the model equals the definition, tests/test_gpu_tsdf_batch.py runs them through the kernel."""
from collections import Counter

import numpy as np

F = np.float32
EPS = F(1e-6)
WEIGHT_PATHS = ("saturated", "wide", "unrolled", "partial", "general")
DISTANCE_PATHS = ("commit", "replay")


def fminf(a, b):
    return a if np.isnan(b) else b if np.isnan(a) else min(a, b)


def fmaxf(a, b):
    return a if np.isnan(b) else b if np.isnan(a) else max(a, b)


def clamp_distance(nd, trunc):
    return fminf(trunc, nd) if nd > 0 else fmaxf(F(-trunc), nd)


def blend_two_colors(c1, w1, c2, w2):
    total = F(w1 + w2)
    w1, w2 = F(w1 / total), F(w2 / total)
    out = 0
    for k in range(4):
        a, b = F((int(c1) >> (8 * k)) & 0xFF), F((int(c2) >> (8 * k)) & 0xFF)
        v = F(F(a * w1) + F(b * w2))
        out |= (int(np.floor(abs(v) + F(0.5))) & 0xFF) << (8 * k)     # roundf: halves away from zero; v >= 0 here
    return out


def sequential(trunc, max_w, sdf, uw, colors, blend, dist, wgt, rgba):
    """n calls of tsdf_chain_step."""
    trunc, max_w, dist, wgt, rgba = F(trunc), F(max_w), F(dist), F(wgt), int(rgba)
    with np.errstate(all="ignore"):
        for k in range(len(sdf)):
            s, u = F(sdf[k]), F(uw[k])
            nw = F(wgt + u)
            if nw < EPS:
                continue
            nd = F(F(F(s * u) + F(dist * wgt)) / nw)
            if blend and abs(s) < trunc:
                rgba = blend_two_colors(rgba, wgt, 0 if colors is None else colors[k], u)
            dist = clamp_distance(nd, trunc)
            wgt = fminf(max_w, nw)
    return dist, wgt, rgba


def butterfly_sum(u32):
    v = u32.astype(F).copy()
    o = 16
    while o > 0:
        v = (v + v[np.arange(32) ^ o]).astype(F)      # usum += __shfl_xor_sync(usum, o)
        o >>= 1
    return v[0]


def one_batch(trunc, max_w, wide, sdf, uw, colors, blend, dist, wgt, rgba):
    """tsdf_batch for one batch (len(sdf) = nb <= 32).  Returns (dist, wgt, rgba, weight path, distance path, moved mask)."""
    nb = len(sdf)
    negative = bool(np.any(~(uw >= 0)))
    before = np.full(nb, wgt, F)
    wc = wgt
    if wgt == max_w and not negative:
        wpath = "saturated"
    else:
        padded = np.zeros(32, F)
        padded[:nb] = uw
        plain = (not negative) and wgt >= EPS and F(F(wgt + butterfly_sum(padded)) * F(1.001)) < max_w
        if plain:
            wpath = ("wide" if wide else "unrolled") if nb == 32 else "partial"
            for j in range(nb):
                before[j] = wc
                wc = F(wc + uw[j])
        else:
            wpath = "general"
            for j in range(nb):
                before[j] = wc
                nw = F(wc + uw[j])
                if not (nw < EPS):
                    wc = fminf(max_w, nw)
    applies = np.zeros(nb, bool)
    dn = np.full(nb, dist, F)
    for j in range(nb):
        nw = F(before[j] + uw[j])
        if not (nw < EPS):
            applies[j] = True
            dn[j] = clamp_distance(F(F(F(sdf[j] * uw[j]) + F(dist * before[j])) / nw), trunc)
    if blend:
        for j in range(nb):
            if applies[j] and abs(sdf[j]) < trunc:
                rgba = blend_two_colors(rgba, before[j], 0 if colors is None else colors[j], uw[j])
    moved = applies & (dn.view(np.uint32) != np.array(dist, F).view(np.uint32))
    dpath = "commit"
    if moved.any():
        dpath = "replay"
        f = int(np.argmax(moved))
        dist = dn[f]
        for j in range(f + 1, nb):
            nw = F(before[j] + uw[j])
            if not (nw < EPS):
                dist = clamp_distance(F(F(F(sdf[j] * uw[j]) + F(dist * before[j])) / nw), trunc)
    return dist, wc, rgba, wpath, dpath, moved


def batch_walk(trunc, max_w, wide, sdf, uw, colors, blend, dist, wgt, rgba):
    """The batch loop of k_voxel_apply_long over n records.  Returns (dist, wgt, rgba, Counter{(weight path, distance path): batches},
    [first mover of every replayed batch as (batch, record)])."""
    trunc, max_w, dist, wgt, rgba = F(trunc), F(max_w), F(dist), F(wgt), int(rgba)
    sdf, uw = np.asarray(sdf, F), np.asarray(uw, F)
    paths, movers = Counter(), []
    with np.errstate(all="ignore"):
        for b, base in enumerate(range(0, len(sdf), 32)):
            sl = slice(base, min(base + 32, len(sdf)))
            dist, wgt, rgba, wp, dp, moved = one_batch(trunc, max_w, wide, sdf[sl], uw[sl], None if colors is None else colors[sl], blend,
                                                       dist, wgt, rgba)
            paths[(wp, dp)] += 1
            if dp == "replay":
                movers.append((b, int(np.argmax(moved))))
    return dist, wgt, rgba, paths, movers


# ---------------------------------------------------------------------------------------------------------------------------
# families
# ---------------------------------------------------------------------------------------------------------------------------
TRUNC = F(0.4)
LENGTHS = (1, 31, 32, 33, 63, 64, 65, 96, 4096, 4097)
MAX_WEIGHTS = (1.0, 3.5, 50.0, 1e4)


def up(x, k=1):
    x = F(x)
    for _ in range(k):
        x = np.nextafter(x, F(np.inf), dtype=F)
    return x


def plain_condition(w, u, max_w):
    padded = np.zeros(32, F)
    padded[:len(u)] = u
    return bool(np.all(u >= 0)) and bool(F(w) >= EPS) and bool(F(F(F(w) + butterfly_sum(padded)) * F(1.001)) < F(max_w))


def margin_pair(rng, nb, max_w, w0):
    """Two weight batches that differ by the last bits of a scale factor: one just takes the bare chain, the other just does not."""
    u = rng.uniform(0.2, 1.0, nb)
    u *= (float(max_w) / 1.001 - float(w0)) / u.sum()
    lo, hi = 0.9, 1.1                                  # plain at lo, refused at hi
    assert plain_condition(w0, (u * lo).astype(F), max_w) and not plain_condition(w0, (u * hi).astype(F), max_w)
    for _ in range(60):
        mid = 0.5 * (lo + hi)
        if plain_condition(w0, (u * mid).astype(F), max_w):
            lo = mid
        else:
            hi = mid
    return (u * lo).astype(F), (u * hi).astype(F)


def families(seed=11):
    """[{name, trunc, max_weight, dist, wgt, rgba, sdf, uw, colors, blend}]"""
    rng = np.random.default_rng(seed)
    out = []

    def fam(name, max_w, w0, d0, sdf, uw, colors=None, blend=False, rgba=0):
        out.append(dict(name=name, trunc=TRUNC, max_weight=F(max_w), dist=F(d0), wgt=F(w0), rgba=int(rgba), sdf=np.asarray(sdf, F),
                        uw=np.asarray(uw, F), colors=None if colors is None else np.asarray(colors, np.uint32), blend=bool(blend)))

    moving = lambda n: rng.uniform(-0.3, 0.3, n)                    # |sdf| < truncation: every record moves the distance
    far = lambda n: rng.uniform(0.8, 3.0, n)                        # sdf > truncation: a voxel at +truncation stays pinned
    # voxel weight at and around the 1e-6 skip threshold; weights with zeros, values below 1e-6, one NaN, one negative
    for tag, w0 in (("zero", 0.0), ("below_eps", 5e-7), ("eps", EPS), ("above_eps", up(EPS))):
        fam(f"start_{tag}_tiny_weights", 50.0, w0, 0.0, moving(64), rng.choice([0.0, 3e-7, 8e-7, 0.5], 64, p=[0.4, 0.25, 0.25, 0.1]))
        uw = rng.uniform(0.0, 0.2, 40)
        uw[5] = np.nan
        fam(f"start_{tag}_one_nan", 50.0, w0, 0.1, moving(40), uw)
        uw = rng.uniform(0.0, 0.2, 64)
        uw[7] = -0.25
        fam(f"start_{tag}_one_negative", 50.0, w0, 0.1, moving(64), uw)
    # saturated voxel
    for max_w in MAX_WEIGHTS:
        fam(f"saturated_pinned_max{max_w:g}", max_w, max_w, TRUNC, far(96), rng.uniform(0.0, 1.0, 96))
        fam(f"saturated_moving_max{max_w:g}", max_w, max_w, 0.1, moving(96), rng.uniform(0.0, 1.0, 96))
        uw = rng.uniform(0.0, 1.0, 96)
        uw[32 + 9] = -0.75 * max_w                                  # the middle batch must not be skipped
        fam(f"saturated_one_negative_max{max_w:g}", max_w, max_w, 0.1, moving(96), uw)
    # the bare chain's bound, a few ulp on either side of max_weight; full batch, partial batch, full + partial
    for max_w in MAX_WEIGHTS:
        for nb in (32, 20):
            below, above = margin_pair(rng, nb, F(max_w), F(0.25 * max_w))
            for tag, u in (("below", below), ("above", above)):
                fam(f"margin_{tag}_nb{nb}_max{max_w:g}", max_w, 0.25 * max_w, TRUNC, far(nb), u)
                fam(f"margin_{tag}_nb{nb}_after_full_batch_max{max_w:g}", max_w, 0.25 * max_w - 0.032 * max_w, 0.05, moving(32 + nb),
                    np.concatenate([np.full(32, 0.001 * max_w), u]))
    # the clamp reached at record k of the second batch, and in the partial last batch
    for max_w in MAX_WEIGHTS:
        for k in (0, 15, 31):
            uw = np.full(32 + 32 + 11, 1e-4 * max_w)
            uw[32 + k] = 0.6 * max_w
            fam(f"clamp_at_record{k}_max{max_w:g}", max_w, 0.5 * max_w, 0.2, moving(75), uw)
        uw = np.full(32 + 11, 1e-4 * max_w)
        uw[32 + 5] = 0.6 * max_w
        fam(f"clamp_in_last_batch_max{max_w:g}", max_w, 0.5 * max_w, TRUNC, far(43), uw)
    # the distance: pinned for the whole chain, first mover at a chosen record, every record moves, sums that cancel
    fam("pinned_plus", 1e4, 3.0, TRUNC, far(150), rng.uniform(0.0, 1.0, 150))
    fam("pinned_minus", 1e4, 3.0, -TRUNC, -far(150), rng.uniform(0.0, 1.0, 150))
    for k in (0, 1, 31, 64 + 3):
        sdf = far(64 + 9)
        sdf[k] = 0.1
        fam(f"first_mover_at_record{k}", 1e4, 3.0, TRUNC, sdf, rng.uniform(0.1, 1.0, 73))
    fam("every_record_moves", 1e4, 3.0, 0.0, moving(130), rng.uniform(0.1, 1.0, 130))
    fam("cancel_to_plus_zero", 1e4, 1.0, 0.25, [-0.25, 0.3, -0.1] * 11, np.ones(33))
    fam("cancel_from_minus_zero", 1e4, 1.0, -0.0, [0.0] * 5 + [-0.0] * 5 + [0.0] * 23, np.ones(33))
    fam("cancel_from_plus_zero", 1e4, 1.0, 0.0, [-0.0] * 40, np.ones(40))
    # chain lengths around the batch size and around the hot-voxel threshold; the long ones cross the clamp on the way
    for n in LENGTHS:
        fam(f"length_{n}_moving", 50.0, 0.5, 0.0, moving(n), rng.uniform(0.0, 0.03, n))
        fam(f"length_{n}_pinned", 50.0, 0.5, TRUNC, far(n), rng.uniform(0.0, 0.03, n))
    # colour blending in record order, only where |sdf| < truncation
    for tag, w0, max_w in (("unsaturated", 2.0, 1e4), ("saturated", 50.0, 50.0), ("crossing", 40.0, 50.0), ("from_zero", 0.0, 50.0)):
        n = 100
        sdf = np.where(rng.random(n) < 0.5, moving(n), far(n))
        fam(f"blend_{tag}", max_w, w0, TRUNC, sdf, rng.uniform(0.0, 0.5, n), colors=rng.integers(0, 1 << 32, n, dtype=np.uint64),
            blend=True, rgba=0x80402010)
        fam(f"blend_{tag}_black_points", max_w, w0, TRUNC, sdf, rng.uniform(0.0, 0.5, n), blend=True, rgba=0xFFC08040)
    return out


def run_family(f, wide, walk=batch_walk):
    return walk(f["trunc"], f["max_weight"], wide, f["sdf"], f["uw"], f["colors"], f["blend"], f["dist"], f["wgt"], f["rgba"])


def run_sequential(f):
    return sequential(f["trunc"], f["max_weight"], f["sdf"], f["uw"], f["colors"], f["blend"], f["dist"], f["wgt"], f["rgba"])


def same_state(a, b):
    return (np.array(a[0], F).tobytes(), np.array(a[1], F).tobytes(), int(a[2])) == \
           (np.array(b[0], F).tobytes(), np.array(b[1], F).tobytes(), int(b[2]))
