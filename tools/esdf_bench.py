"""Cost of the batch ESDF (ksg_compute_esdf) of bench.py's `fast5` map.

  python tools/esdf_bench.py [--frames 300] [--reps 5] [--json OUT]

Builds the map from the first --frames frames of bench.py's synthetic 640x480 stream (5 cm voxels, C = 21, `fast`), then at
max_distance 1.0 and 2.0 m reports:
  - the host wall time of ksg_compute_esdf with distance and flags into host arrays (median of --reps calls after one warm-up);
  - the device time of each of its kernels, from a separate torch.profiler run (CUDA activities) of --reps calls;
  - the three work-set sizes in blocks (x pass, y pass, z pass = the allocated blocks), counted on the host from the exported map by
    the rule of csrc/ksg_esdf.cuh, with the surface blocks taken from the call's own flags;
  - the share of observed voxels that are CAPPED.
Prints one JSON object with the card's name and power limit."""
import argparse
import json
import math
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from bench import WORKLOADS, gen_frames, gpu_identity, make_cfg  # noqa: E402
from kimera_semantics_b200.capi import KSG_ESDF_CAPPED, KSG_ESDF_OBSERVED, KSG_ESDF_SURFACE, Integrator  # noqa: E402


def work_sets(block_index, site_blocks, Rb):
    """sizes of the x- and y-pass work sets (ksg_esdf.cuh): Y = within Rb along z of an allocated block with a near-x block within Rb
    along y; X = within Rb along y of a Y block and near-x; near-x = within Rb along x of a block holding a site"""
    near_x = {(b[0] + k, b[1], b[2]) for b in map(tuple, block_index[site_blocks].tolist()) for k in range(-Rb, Rb + 1)}
    cand = {(b[0], b[1], b[2] + k) for b in map(tuple, block_index.tolist()) for k in range(-Rb, Rb + 1)}
    ys = {b for b in cand if any((b[0], b[1] + j, b[2]) in near_x for j in range(-Rb, Rb + 1))}
    xs = {(b[0], b[1] + j, b[2]) for b in ys for j in range(-Rb, Rb + 1)} & near_x
    return len(xs), len(ys)


def kernel_name(key):
    if "k_esdf_sites" in key:
        return "k_esdf_sites"
    for a in "012":
        if f"k_esdf_pass<{a}" in key or f"k_esdf_passILi{a}E" in key:
            return f"k_esdf_pass<{a}>"
    return key


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--frames", type=int, default=300)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--json", default=None, help="also write the result to this file")
    args = ap.parse_args()

    workload = "fast5"
    _, w, h, vs, _, _, _ = WORKLOADS[workload]
    cfg = make_cfg(workload)
    vps = cfg.voxels_per_side
    cam, frames = gen_frames(workload, args.frames)
    integ = Integrator(cfg)
    stream = torch.cuda.Stream()
    with torch.cuda.stream(stream):
        for depth, label, T in frames:
            d_depth, d_label = torch.from_numpy(depth).cuda(), torch.from_numpy(label).cuda()
            integ.integrate_depth_device(T, d_depth.data_ptr(), d_label.data_ptr(), w, h, cam.K, stream=stream.cuda_stream)
    stream.synchronize()
    integ.sync()
    res = {"workload": workload, "frames": args.frames, "blocks": integ.num_blocks(), "voxels_per_side": vps, "voxel_size_m": vs,
           "gpu": gpu_identity(0), "max_distance": {}}
    for m in (1.0, 2.0):
        W = int(math.ceil(float(np.float32(m)) / float(np.float32(vs)))) + 1
        Rb = -(-W // vps)
        out = integ.esdf(m)                                          # warm-up
        wall = []
        for _ in range(args.reps):
            t0 = time.perf_counter()
            out = integ.esdf(m)
            wall.append(time.perf_counter() - t0)
        fl = out["flags"]
        observed = (fl & KSG_ESDF_OBSERVED) != 0
        site_blocks = ((fl & KSG_ESDF_SURFACE) != 0).any(axis=1)
        n_x, n_y = work_sets(out["block_index"], site_blocks, Rb)
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            for _ in range(args.reps):
                integ.esdf(m)
            torch.cuda.synchronize()
        kernels = {}
        for e in prof.key_averages():
            if "esdf" in e.key:
                kernels[kernel_name(e.key)] = {"us_per_call": e.device_time_total / max(e.count, 1), "calls": e.count}
        res["max_distance"][str(m)] = {
            "window_voxels": W, "window_blocks": Rb,
            "host_wall_ms": {"median": 1e3 * float(np.median(wall)), "min": 1e3 * min(wall), "max": 1e3 * max(wall)},
            "device_us": kernels,
            "work_set_blocks": {"x_pass": n_x, "y_pass": n_y, "z_pass": int(len(fl))},
            "site_blocks": int(site_blocks.sum()),
            "share_capped_of_observed": float(((fl & KSG_ESDF_CAPPED) != 0).sum() / max(int(observed.sum()), 1)),
            "observed_voxels": int(observed.sum())}
    integ.close()
    print(json.dumps(res))
    if args.json:
        with open(args.json, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
