"""Cost of keeping the semantic mesh on the device (ksg_update_mesh) while the map grows, against one whole-map ksg_extract_mesh.

  python tools/mesh_incremental_bench.py [--frames 300] [--start 100] [--maps fast5,fast2cm] [--json OUT]

The two maps of tools/esdf_incremental_bench.py: bench.py's synthetic 640x480 `fast` stream (C = 21) at 5 cm (`fast5`, max_blocks 8192)
and at 2 cm (`fast2cm`, max_blocks 32768).  For each map, an update (min_weight 1e-4) after every frame and after every 10th from frame
--start on:
  - host wall time of each update (the frame's stream is synchronised first, so the time is the update's alone): median and max over
    the incremental updates, and the first (full) update apart;
  - remeshed_blocks / blocks, remeshed_vertices and the layer's vertices over the incremental updates, median and max;
  - from a separate torch.profiler run of the same sequence: device time per kernel and per update, and memcpy / memset time;
  - one whole-map ksg_extract_mesh on the final map: host wall time (median of 3) and device time of its kernels.
Prints one JSON object with the card's name and power limit."""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from bench import gen_frames, gpu_identity, make_cfg  # noqa: E402
from esdf_incremental_bench import MAPS, is_cuda, stats_of  # noqa: E402
from kimera_semantics_b200.capi import Integrator  # noqa: E402

KERNELS = ("k_mesh_dirty", "k_mesh_scan", "k_mesh_move", "k_mesh_blocks<false>", "k_mesh_blocks<true>")


def kernel_name(key):
    if "k_mesh_blocks" in key:
        return "k_mesh_blocks<true>" if ("ILb1E" in key or "<true>" in key) else "k_mesh_blocks<false>"
    for k in KERNELS:
        if k in key:
            return k
    return key


def split(prof, label):
    """per range `label`: ({kernel: us}, copy us) of the device work inside it"""
    evs = prof.events()
    ranges = sorted((e.time_range.start, e.time_range.end) for e in evs if e.name == label and not is_cuda(e))
    per = [({}, 0.0) for _ in ranges]
    starts = np.array([r[0] for r in ranges])
    for e in evs:
        if not is_cuda(e) or e.name == label:
            continue
        i = int(np.searchsorted(starts, e.time_range.start, side="right")) - 1
        if i < 0 or e.time_range.end > ranges[i][1]:
            continue
        us = e.time_range.end - e.time_range.start
        if "emcpy" in e.name or "emset" in e.name:
            per[i] = (per[i][0], per[i][1] + us)
        elif "k_mesh" in e.name:
            k = kernel_name(e.name)
            per[i][0][k] = per[i][0].get(k, 0.0) + us
    return per


def run(cfg, dev_frames, cam, w, h, every, start, profile):
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
            with torch.profiler.record_function("mesh_update"):
                st = integ.update_mesh()
            updates.append((0.0, st))
        else:
            t0 = time.perf_counter()
            st = integ.update_mesh()
            updates.append((time.perf_counter() - t0, st))
    stream.synchronize()
    if prof:
        prof.__exit__(None, None, None)
    return integ, updates, prof


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
        out = {"voxel_size_m": vs, "max_blocks": max_blocks}
        for every in (1, 10):
            integ, ups, _ = run(cfg, dev_frames, cam, w, h, every, args.start, False)
            inc = [u for u in ups if not u[1]["full"]]
            walls = [1e3 * u[0] for u in inc]
            r = {"updates": len(ups), "first_full_ms": 1e3 * ups[0][0], "blocks_final": ups[-1][1]["blocks"],
                 "vertices_final": ups[-1][1]["vertices"], "wall_ms": stats_of(walls),
                 "remeshed_over_blocks": stats_of([u[1]["remeshed_blocks"] / max(u[1]["blocks"], 1) for u in inc]),
                 "changed_blocks": stats_of([u[1]["changed_blocks"] for u in inc]),
                 "remeshed_blocks": stats_of([u[1]["remeshed_blocks"] for u in inc]),
                 "remeshed_vertices": stats_of([u[1]["remeshed_vertices"] for u in inc]),
                 "vertices": stats_of([u[1]["vertices"] for u in inc])}
            if every == 1:                                                # the whole-map batch entry on the final map
                integ.extract_mesh()
                bw = []
                for _ in range(3):
                    t0 = time.perf_counter()
                    integ.extract_mesh()
                    bw.append(1e3 * (time.perf_counter() - t0))
                with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CPU, torch.profiler.ProfilerActivity.CUDA]) as bp:
                    for _ in range(3):
                        with torch.profiler.record_function("mesh_batch"):
                            integ.extract_mesh()
                bs = split(bp, "mesh_batch")
                out["extract_mesh_final_map"] = {"blocks": integ.num_blocks(), "wall_ms": float(np.median(bw)),
                                                 "kernel_us": float(np.median([sum(k.values()) for k, _ in bs])),
                                                 "copy_us": float(np.median([c for _, c in bs]))}
            integ.close()
            integ, _, prof = run(cfg, dev_frames, cam, w, h, every, args.start, True)
            integ.close()
            sp = split(prof, "mesh_update")[1:]                           # the incremental updates
            names = sorted({n for k, _ in sp for n in k})
            r["device_us_per_update"] = {n: stats_of([k.get(n, 0.0) for k, _ in sp]) for n in names}
            r["kernel_us"] = stats_of([sum(k.values()) for k, _ in sp])
            r["copy_us"] = stats_of([c for _, c in sp])
            out[f"every_{every}"] = r
        res["maps"][name] = out
    print(json.dumps(res))
    if args.json:
        with open(args.json, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
