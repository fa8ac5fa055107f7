"""Where the fast integrator's persistent solve kernel (k_fast_solve3) spends a frame, phase by phase, without perturbing it.

  python tools/solver_phases.py [--workload fast5] [--frames 200] [--warmup 20] [--json OUT]

Runs bench.py's frames of the workload through capi.Integrator with profiling on and KSG_PROFILE_MARKS_ONLY=1: block 0 of the
solve kernel stamps clock64 at every grid-wide phase boundary, and the per-ray probes of the full profiling mode (same-address
atomics that slow the ray set-up most) stay off.  Prints the median over the frames of every phase in microseconds, the front
(everything before the first sweep), the sweeps and the tail (everything after the last sweep), with the card's name and power
limit.  Microseconds are clock64 ticks over the device's nominal SM clock; under a lower clock the shares stay right.
"""
import argparse
import ctypes as C
import json
import os
import sys

import numpy as np

os.environ["KSG_PROFILE_MARKS_ONLY"] = "1"   # read when the integrator is created
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from bench import WORKLOADS, gen_frames, gpu_identity, make_cfg  # noqa: E402


def phases(tl, sweeps, khz):
    """Phase spans (µs) of one frame from the raw timeline slots of ksg_debug_fast_timeline."""
    us = lambda a, b: (tl[b] - tl[a]) / (khz / 1e3)
    tb = 52                                   # kTimelineSlots - 12: first mark after the sweeps
    return {"front": us(0, 2), "ray_setup": us(1, 2), "before_ray_setup": us(0, 1),
           "sweeps": us(2, 2 + sweeps), "first_sweep": us(2, 3),
           "commit_alloc_count": us(tb, tb + 1), "tile_alloc_block_init": us(tb + 2, tb + 3), "scatter": us(tb + 3, tb + 4),
           "tail": us(2 + sweeps, tb + 4), "kernel": us(0, tb + 4)}


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--workload", default="fast5", choices=[k for k, v in WORKLOADS.items() if k.startswith("fast")])
    ap.add_argument("--frames", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--json", default=None, help="also write the per-frame phases and medians to this file")
    args = ap.parse_args()

    import torch
    from kimera_semantics_b200.capi import Integrator
    _, w, h, _, _, _, _ = WORKLOADS[args.workload]
    n = args.warmup + args.frames
    cam, frames = gen_frames(args.workload, n)
    d_depth = [torch.from_numpy(f[0]).cuda() for f in frames]
    d_label = [torch.from_numpy(f[1]).cuda() for f in frames]
    integ = Integrator(make_cfg(args.workload))
    ts = torch.cuda.Stream()
    torch.cuda.set_stream(ts)
    for i in range(args.warmup):
        integ.integrate_depth_device(frames[i][2], d_depth[i].data_ptr(), d_label[i].data_ptr(), w, h, cam.K, ts.cuda_stream)
    integ.sync()
    integ.set_profiling(True)
    out64 = (C.c_int64 * 80)()
    per_frame, sweeps = [], []
    for i in range(args.warmup, n):
        integ.integrate_depth_device(frames[i][2], d_depth[i].data_ptr(), d_label[i].data_ptr(), w, h, cam.K, ts.cuda_stream)
        ns, khz = C.c_int64(), C.c_double()
        if int(integ.lib.ksg_debug_fast_timeline(integ.handle, out64, C.byref(ns), C.byref(khz))) == 0:
            raise SystemExit("no solve-kernel timeline: is this the fast integrator?")
        per_frame.append(phases([int(v) for v in out64], int(ns.value), khz.value))
        sweeps.append(int(ns.value))
    prof = integ.get_profile()
    integ.close()

    med = {k: float(np.median([p[k] for p in per_frame])) for k in per_frame[0]}
    gpu = gpu_identity(0)
    print(f"{args.workload}: {args.frames} frames after {args.warmup} warm-up frames; {gpu}")
    print(f"sweeps per frame: median {int(np.median(sweeps))}, range {min(sweeps)}-{max(sweeps)}")
    print("median per phase (µs at the nominal SM clock, share of the solve kernel):")
    for k in ("before_ray_setup", "ray_setup", "front", "first_sweep", "sweeps", "commit_alloc_count", "tile_alloc_block_init", "scatter",
              "tail", "kernel"):
        print(f"  {k:24s} {med[k]:8.1f}  {100.0 * med[k] / med['kernel']:5.1f} %")
    frame_us = 1e3 * prof["frame"] / max(1, prof["frames"])
    print(f"frame (CUDA events, mean): {frame_us:.1f} µs; front + tail = {100.0 * (med['front'] + med['tail']) / frame_us:.1f} % of it")
    if args.json:
        with open(args.json, "w") as fh:
            json.dump({"workload": args.workload, "gpu": gpu, "median_us": med, "frame_us": frame_us, "sweeps": sweeps, "frames": per_frame}, fh)


if __name__ == "__main__":
    main()
