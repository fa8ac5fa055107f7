"""Cost of keeping the ESDF on the device (ksg_update_esdf) while the map grows, against one batch ksg_compute_esdf.

  python tools/esdf_incremental_bench.py [--frames 300] [--start 100] [--json OUT]

Two maps of bench.py's synthetic 640x480 stream (`fast`, C = 21): `fast5` (5 cm voxels, max_blocks 8192, as bench.py runs it) and
`fast2cm` (the same stream at 2 cm with merged2's max_blocks, 32768).  For each map, max_distance 1.0 and 2.0 m and an update after
every frame and after every 10th from frame --start on:
  - host wall time of each update (the frame's stream is synchronised first, so the time is the update's alone): median and max over
    the incremental updates, and the first (full) update apart;
  - the stats of every incremental update: z_blocks / blocks, x_blocks and y_blocks, median and max;
  - from a separate torch.profiler run of the same sequence: device time per kernel and per update, memcpy / memset time per update, and
    the wall-time split of the median update into kernels, copies and host (the rest);
  - a batch ksg_compute_esdf on the final map: host wall time (median of 3) and device time of its kernels.
Prints one JSON object with the card's name and power limit."""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from bench import gen_frames, gpu_identity, make_cfg  # noqa: E402
from kimera_semantics_b200.capi import Integrator  # noqa: E402

MAPS = {"fast5": (0.05, 8192), "fast2cm": (0.02, 32768)}


def kernel_name(key):
    for k in ("k_esdf_sites", "k_esdf_gather", "k_query_esdf"):
        if k in key:
            return k
    for a in "012":
        if f"k_esdf_pass<{a}" in key or f"k_esdf_passILi{a}E" in key:
            return f"k_esdf_pass<{a}>"
    return key


def is_cuda(e):
    return str(getattr(e, "device_type", "")).endswith("CUDA")


def run(cfg, dev_frames, cam, w, h, m, every, start, profile):
    """integrate the stream, updating the layer every `every` frames from `start` on: (integrator, [(wall s, stats)], profiler or None)"""
    integ = Integrator(cfg)
    stream = torch.cuda.Stream()
    updates = []
    prof = torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CPU, torch.profiler.ProfilerActivity.CUDA]) if profile else None
    if prof:
        prof.__enter__()
    for f, (d_depth, d_label, T) in enumerate(dev_frames):
        with torch.cuda.stream(stream):
            integ.integrate_depth_device(T, d_depth.data_ptr(), d_label.data_ptr(), w, h, cam.K, stream=stream.cuda_stream)
        if f < start or (f - start) % every != 0:
            continue
        stream.synchronize()
        integ.sync()
        if prof:
            with torch.profiler.record_function("esdf_update"):
                st = integ.update_esdf(m)
            updates.append((0.0, st))
        else:
            t0 = time.perf_counter()
            st = integ.update_esdf(m)
            updates.append((time.perf_counter() - t0, st))
    stream.synchronize()
    if prof:
        prof.__exit__(None, None, None)
    return integ, updates, prof


def split(prof, label):
    """per range `label`: ({kernel: us}, copy us) of the device work inside it"""
    evs = prof.events()
    ranges = sorted((e.time_range.start, e.time_range.end) for e in evs if e.name == label and not is_cuda(e))
    per = [({}, 0.0) for _ in ranges]
    starts = np.array([r[0] for r in ranges])
    for e in evs:
        if not is_cuda(e) or e.name == label:                            # the range's own device-side marker is not work
            continue
        i = int(np.searchsorted(starts, e.time_range.start, side="right")) - 1
        if i < 0 or e.time_range.end > ranges[i][1]:
            continue
        us = e.time_range.end - e.time_range.start
        if "Memcpy" in e.name or "Memset" in e.name or "memcpy" in e.name or "memset" in e.name:
            per[i] = (per[i][0], per[i][1] + us)
        elif "esdf" in e.name:
            k = kernel_name(e.name)
            per[i][0][k] = per[i][0].get(k, 0.0) + us
    return per


def stats_of(x):
    return {"median": float(np.median(x)), "max": float(np.max(x))} if len(x) else None


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--frames", type=int, default=300)
    ap.add_argument("--start", type=int, default=100)
    ap.add_argument("--maps", default="fast5,fast2cm")
    ap.add_argument("--json", default=None, help="also write the result to this file")
    args = ap.parse_args()

    cam, frames = gen_frames("fast5", args.frames)
    w, h = cam.width, cam.height
    dev_frames = [(torch.from_numpy(d).cuda(), torch.from_numpy(l).cuda(), T) for d, l, T in frames]
    res = {"frames": args.frames, "start": args.start, "gpu": gpu_identity(0), "maps": {}}
    for name in args.maps.split(","):
        vs, max_blocks = MAPS[name]
        cfg = make_cfg("fast5")
        cfg.voxel_size = vs
        cfg.max_blocks = max_blocks
        out = {"voxel_size_m": vs, "max_blocks": max_blocks, "max_distance": {}}
        for m in (1.0, 2.0):
            per_m = {}
            for every in (1, 10):
                integ, ups, _ = run(cfg, dev_frames, cam, w, h, m, every, args.start, False)
                inc = [u for u in ups if not u[1]["full"]]
                walls = [1e3 * u[0] for u in inc]
                zs = [u[1]["z_blocks"] / max(u[1]["blocks"], 1) for u in inc]
                r = {"updates": len(ups), "first_full_ms": 1e3 * ups[0][0], "blocks_final": ups[-1][1]["blocks"],
                     "wall_ms": stats_of(walls), "z_over_blocks": stats_of(zs),
                     "z_blocks": stats_of([u[1]["z_blocks"] for u in inc]), "x_blocks": stats_of([u[1]["x_blocks"] for u in inc]),
                     "y_blocks": stats_of([u[1]["y_blocks"] for u in inc]),
                     "changed_blocks": stats_of([u[1]["changed_blocks"] for u in inc]),
                     "site_changed": stats_of([u[1]["site_changed"] for u in inc]),
                     "no_change_updates": sum(1 for u in inc if u[1]["changed_blocks"] == 0)}
                if every == 1:                                            # batch on the final map
                    integ.esdf(m)
                    bw = []
                    for _ in range(3):
                        t0 = time.perf_counter()
                        integ.esdf(m)
                        bw.append(1e3 * (time.perf_counter() - t0))
                    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CPU, torch.profiler.ProfilerActivity.CUDA]) as bp:
                        for _ in range(3):
                            with torch.profiler.record_function("esdf_batch"):
                                integ.esdf(m)
                    bs = split(bp, "esdf_batch")
                    per_m["batch_final_map"] = {"blocks": integ.num_blocks(), "wall_ms": float(np.median(bw)),
                                                "kernel_us": float(np.median([sum(k.values()) for k, _ in bs])),
                                                "copy_us": float(np.median([c for _, c in bs]))}
                integ.close()
                integ, _, prof = run(cfg, dev_frames, cam, w, h, m, every, args.start, True)
                integ.close()
                sp = split(prof, "esdf_update")[1:]                       # the incremental updates
                ker = [sum(k.values()) for k, _ in sp]
                cpy = [c for _, c in sp]
                names = sorted({n for k, _ in sp for n in k})
                r["device_us_per_update"] = {n: stats_of([k.get(n, 0.0) for k, _ in sp]) for n in names}
                r["kernel_us"] = stats_of(ker)
                r["copy_us"] = stats_of(cpy)
                if walls:
                    kmed, cmed = float(np.median(ker)) if ker else 0.0, float(np.median(cpy)) if cpy else 0.0
                    wmed = 1e3 * float(np.median(walls))
                    r["wall_split_us"] = {"wall": wmed, "kernels": kmed, "copies": cmed, "host": wmed - kmed - cmed}
                per_m[f"every_{every}"] = r
            out["max_distance"][str(m)] = per_m
        res["maps"][name] = out
    print(json.dumps(res))
    if args.json:
        with open(args.json, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
