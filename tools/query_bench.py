"""Throughput of the point queries (ksg_query_points_device) on bench.py's `fast5` map, against the only way to read the map before
them: exporting every block.

  python tools/query_bench.py [--frames 300] [--passes 5] [--window 0.3] [--json OUT]

Builds the map from the first --frames frames of bench.py's synthetic 640x480 stream (5 cm voxels, C = 21, `fast`), then times with CUDA
events, per point distribution (uniform over the map's bounding box; near the surface = the back-projected pixels of 8 frames,
resampled and jittered by up to +-2 voxels per axis) and count (2^20, 2^24): every output, and every output but the log-probability
rows.  Each figure is the median of --passes passes of at least --window seconds each, after a warm-up.  In the same run: host wall
time of ksg_export_blocks of the whole map (into preallocated host arrays) and of the host entry ksg_query_points on 2^16 points.
Prints one JSON object with queries/s, the bytes a valid query has to read and write, and the card's name and power limit."""
import argparse
import ctypes as C
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
from kimera_semantics_b200 import synth  # noqa: E402
from kimera_semantics_b200.capi import QUERY_FIELDS, Integrator, _ptr  # noqa: E402


def quat_matrix(q):
    w, x, y, z = (float(v) for v in q)
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)],
                     [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
                     [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]])


def surface_points(cam, frames, n_frames):
    """world-frame back-projected pixels of n_frames frames spread over the stream"""
    pts = []
    for depth, _, T in frames[:: max(1, len(frames) // n_frames)][:n_frames]:
        xyz, _ = synth.backproject(depth, cam)
        pts.append(xyz.astype(np.float64) @ quat_matrix(T[:4]).T + np.asarray(T[4:], np.float64))
    return np.concatenate(pts).astype(np.float32)


def device_outputs(n, nl):
    f32, u8 = torch.float32, torch.uint8
    shapes = {"flags": ((n,), u8), "tsdf_distance": ((n,), f32), "tsdf_weight": ((n,), f32), "tsdf_rgba": ((n, 4), u8),
              "sem_label": ((n,), u8), "sem_priors": ((n, nl), f32), "sem_rgba": ((n, 4), u8), "distance": ((n,), f32),
              "gradient": ((n, 3), f32)}
    return {k: torch.empty(s, dtype=t, device="cuda") for k, (s, t) in shapes.items()}


def time_queries(integ, d_xyz, n, ptrs, stream, passes, window):
    """median queries/s over `passes` windows of >= `window` s (CUDA events around back-to-back launches on one stream)"""
    def run(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        for _ in range(reps):
            integ.query_points_device(d_xyz.data_ptr(), n, ptrs, stream=stream.cuda_stream)
        e1.record(stream)
        e1.synchronize()
        return e0.elapsed_time(e1) * 1e-3
    run(3)                                                          # warm-up
    reps = max(1, math.ceil(window / max(run(1), 1e-6)))
    rates = []
    for _ in range(passes):
        t = run(reps)
        rates.append(n * reps / t)
    return {"queries_per_s": float(np.median(rates)), "spread": [float(min(rates)), float(max(rates))], "launches_per_pass": reps}


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--frames", type=int, default=300)
    ap.add_argument("--passes", type=int, default=5)
    ap.add_argument("--window", type=float, default=0.3)
    ap.add_argument("--json", default=None, help="also write the result to this file")
    args = ap.parse_args()

    workload = "fast5"
    _, w, h, vs, nl, _, _ = WORKLOADS[workload]
    cam, frames = gen_frames(workload, args.frames)
    integ = Integrator(make_cfg(workload))
    stream = torch.cuda.Stream()
    with torch.cuda.stream(stream):
        for depth, label, T in frames:
            d_depth, d_label = torch.from_numpy(depth).cuda(), torch.from_numpy(label).cuda()
            integ.integrate_depth_device(T, d_depth.data_ptr(), d_label.data_ptr(), w, h, cam.K, stream=stream.cuda_stream)
    stream.synchronize()
    integ.sync()
    nb = integ.num_blocks()
    vps = integ.cfg.voxels_per_side
    V = vps ** 3

    # whole-map export into preallocated host arrays
    bidx = np.zeros((nb, 3), np.int32)
    arrs = [np.zeros(nb * V, np.float32), np.zeros(nb * V, np.float32), np.zeros(nb * V * 4, np.uint8), np.zeros(nb * V, np.uint8),
            np.zeros(nb * V * nl, np.float32), np.zeros(nb * V * 4, np.uint8)]
    types = [C.c_float, C.c_float, C.c_uint8, C.c_uint8, C.c_float, C.c_uint8]
    export_s = []
    for _ in range(args.passes + 1):
        t0 = time.perf_counter()
        rc = integ.lib.ksg_export_blocks(integ.handle, nb, _ptr(bidx, C.c_int32), *[_ptr(a, t) for a, t in zip(arrs, types)])
        export_s.append(time.perf_counter() - t0)
        assert rc == 0, rc
    export_bytes = sum(a.nbytes for a in arrs) + bidx.nbytes

    lo = (bidx.min(axis=0).astype(np.float64)) * vps * vs
    hi = (bidx.max(axis=0).astype(np.float64) + 1) * vps * vs
    surf = torch.from_numpy(surface_points(cam, frames, 8)).cuda()
    gen = torch.Generator(device="cuda").manual_seed(0)
    res = {"workload": workload, "frames": args.frames, "blocks": nb, "gpu": gpu_identity(0),
           "map_box_m": [lo.tolist(), hi.tolist()],
           "export_blocks_whole_map_s": float(np.median(export_s[1:])), "export_bytes": int(export_bytes)}
    # bytes of a valid query: point, containing voxel (distance, weight, colour, semantic colour, label), the 32 distinct voxels
    # (distance + weight) of the gradient's 6 trilinear stencils (D(p) is inside them), the row when wanted; hash probes not counted
    res["bytes_read_per_query"] = {"with_rows": 12 + 17 + 32 * 8 + 4 * nl, "without_rows": 12 + 17 + 32 * 8}
    res["bytes_written_per_query"] = {"with_rows": 1 + 4 + 4 + 4 + 1 + 4 + 4 + 12 + 4 * nl, "without_rows": 1 + 4 + 4 + 4 + 1 + 4 + 4 + 12}
    runs = {}
    for lg in (20, 24):
        n = 1 << lg
        box_lo, box_hi = torch.tensor(lo, dtype=torch.float32, device="cuda"), torch.tensor(hi, dtype=torch.float32, device="cuda")
        uni = box_lo + torch.rand((n, 3), generator=gen, device="cuda") * (box_hi - box_lo)
        pick = torch.randint(0, len(surf), (n,), generator=gen, device="cuda")
        near = surf[pick] + (torch.rand((n, 3), generator=gen, device="cuda") * 4.0 - 2.0) * vs
        out = device_outputs(n, nl)
        torch.cuda.synchronize()
        for dist, d_xyz in (("uniform", uni.contiguous()), ("near_surface", near.contiguous())):
            for rows in (True, False):
                ptrs = {k: out[k].data_ptr() for k in QUERY_FIELDS if rows or k != "sem_priors"}
                r = time_queries(integ, d_xyz, n, ptrs, stream, args.passes, args.window)
                fl = out["flags"].cpu().numpy()
                r["share_interpolated"] = float(((fl & 4) != 0).mean())
                r["share_gradient"] = float(((fl & 8) != 0).mean())
                runs[f"{dist}_2^{lg}_{'with' if rows else 'without'}_rows"] = r
        del out, uni, near
        torch.cuda.empty_cache()
    res["device_queries"] = runs
    # host entry on 2^16 points near the surface
    n = 1 << 16
    hp = (surf[torch.randint(0, len(surf), (n,), generator=gen, device="cuda")]).cpu().numpy()
    integ.query_points(hp)
    host_s = []
    for _ in range(args.passes):
        t0 = time.perf_counter()
        integ.query_points(hp)
        host_s.append(time.perf_counter() - t0)
    res["host_entry_2^16_s"] = float(np.median(host_s))
    integ.close()
    print(json.dumps(res))
    if args.json:
        with open(args.json, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
