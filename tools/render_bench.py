"""Time of a 640x480 render of bench.py's `fast5` map (ksg_render_view_device / ksg_render_view) from poses the map never saw.

  python tools/render_bench.py [--frames 300] [--held-out 4] [--passes 5] [--window 0.3] [--json OUT]

Builds the map from the first --frames frames of bench.py's synthetic 640x480 stream (5 cm voxels, C = 21, `fast`) and renders at
640x480 from the poses of the next --held-out frames of that stream (not integrated), min_depth 0.1 m, max_depth 6 m.  Timed with CUDA
events around back-to-back device renders on one stream, cycling through the held-out poses; each figure is the median of --passes
passes of at least --window seconds each, after a warm-up:
  - depth only (one launch);
  - depth + points + label + gradient (the march, then the point query at the hits);
  - every output, the log-probability rows included.
In the same run: host wall time of the host entry (depth + label + gradient into host arrays), the share of pixels hit, and the
samples per ray counted by the numpy twin (tests/render_ref.py) on every 7th pixel of the first held-out pose.  Prints one JSON object
with the card's name and power limit."""
import argparse
import json
import math
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from bench import WORKLOADS, gen_frames, gpu_identity, make_cfg  # noqa: E402
from kimera_semantics_b200.capi import Integrator  # noqa: E402

MIN_DEPTH, MAX_DEPTH = 0.1, 6.0


def device_outputs(n, nl):
    f32, u8 = torch.float32, torch.uint8
    shapes = {"depth": ((n,), f32), "points_G": ((n, 3), f32), "flags": ((n,), u8), "tsdf_distance": ((n,), f32),
              "tsdf_weight": ((n,), f32), "tsdf_rgba": ((n, 4), u8), "sem_label": ((n,), u8), "sem_priors": ((n, nl), f32),
              "sem_rgba": ((n, 4), u8), "distance": ((n,), f32), "gradient": ((n, 3), f32)}
    return {k: torch.empty(s, dtype=t, device="cuda") for k, (s, t) in shapes.items()}


def time_renders(integ, poses, K, w, h, ptrs, stream, passes, window):
    """median renders/s over `passes` windows of >= `window` s (CUDA events around back-to-back renders on one stream)"""
    def run(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        for i in range(reps):
            integ.render_device(poses[i % len(poses)], K, w, h, MIN_DEPTH, MAX_DEPTH, ptrs, stream=stream.cuda_stream)
        e1.record(stream)
        e1.synchronize()
        return e0.elapsed_time(e1) * 1e-3
    run(2 * len(poses))                                             # warm-up
    reps = max(len(poses), math.ceil(window / max(run(len(poses)) / len(poses), 1e-6)))
    times = [run(reps) / reps for _ in range(passes)]
    return {"ms_per_render": 1e3 * float(np.median(times)), "spread_ms": [1e3 * min(times), 1e3 * max(times)], "renders_per_pass": reps}


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--frames", type=int, default=300)
    ap.add_argument("--held-out", type=int, default=4)
    ap.add_argument("--passes", type=int, default=5)
    ap.add_argument("--window", type=float, default=0.3)
    ap.add_argument("--json", default=None, help="also write the result to this file")
    args = ap.parse_args()

    workload = "fast5"
    _, w, h, vs, nl, _, _ = WORKLOADS[workload]
    cam, frames = gen_frames(workload, args.frames + args.held_out)
    poses = [T for _, _, T in frames[args.frames:]]
    integ = Integrator(make_cfg(workload))
    stream = torch.cuda.Stream()
    with torch.cuda.stream(stream):
        for depth, label, T in frames[:args.frames]:
            d_depth, d_label = torch.from_numpy(depth).cuda(), torch.from_numpy(label).cuda()
            integ.integrate_depth_device(T, d_depth.data_ptr(), d_label.data_ptr(), w, h, cam.K, stream=stream.cuda_stream)
    stream.synchronize()
    integ.sync()
    K = np.array([cam.fx, cam.fy, cam.cx, cam.cy], np.float64)
    n = w * h
    out = device_outputs(n, nl)
    torch.cuda.synchronize()
    res = {"workload": workload, "frames": args.frames, "held_out_poses": len(poses), "blocks": integ.num_blocks(), "image": [w, h],
           "depth_range_m": [MIN_DEPTH, MAX_DEPTH], "gpu": gpu_identity(0)}
    sets = {"depth": ("depth",),
            "depth_label_gradient": ("depth", "points_G", "sem_label", "gradient"),
            "everything_with_rows": tuple(out)}
    runs = {}
    for name, keys in sets.items():
        runs[name] = time_renders(integ, poses, K, w, h, {k: out[k].data_ptr() for k in keys}, stream, args.passes, args.window)
    res["device_render"] = runs
    hit = ~torch.isnan(out["depth"])
    res["share_hit_last_pose"] = float(hit.float().mean())
    # host entry: depth + label + gradient into host arrays
    integ.render(poses[0], K, w, h, MIN_DEPTH, MAX_DEPTH, fields=("depth", "sem_label", "gradient"))
    host_s = []
    for i in range(args.passes):
        t0 = time.perf_counter()
        integ.render(poses[i % len(poses)], K, w, h, MIN_DEPTH, MAX_DEPTH, fields=("depth", "sem_label", "gradient"))
        host_s.append(time.perf_counter() - t0)
    res["host_entry_depth_label_gradient_s"] = float(np.median(host_s))
    # samples per ray, counted by the twin on a subset of the pixels of the first held-out pose
    import render_ref as rr
    exp = integ.export()
    integ.close()
    depth, samples = rr.march(exp, vs, make_cfg(workload).voxels_per_side, poses[0], K, w, h, MIN_DEPTH, MAX_DEPTH,
                              pixels=np.arange(0, n, 7))
    s = samples[::7]
    res["samples_per_ray_twin"] = {"pixels": int(len(s)), "mean": float(s.mean()), "max": int(s.max()),
                                   "share_hit": float((~np.isnan(depth[::7])).mean())}
    print(json.dumps(res))
    if args.json:
        with open(args.json, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
