"""Device time of every launch and memset of a `fast` frame, from a torch.profiler trace (CUDA activities).

  python tools/frame_kernels.py [--workload fast5] [--frames 50] [--warmup 20] [--trace OUT.json]

Runs bench.py's frames of the workload through capi.Integrator on a torch stream, device-resident input, no statistics read per
frame (as bench.py's `value` leg does), traces the timed frames and prints per kernel / memset: calls per frame, mean device µs per
frame and its share of the frame, then the busy time, the span from the first launch's start to the last one's end over the frames,
and what is left of the span (gaps between launches), with the card's name and power limit.  The trace itself slows the host, so
the span here is not bench.py's frame time; the device time of each kernel is.
"""
import argparse
import json
import os
import sys
import tempfile
from collections import defaultdict

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from bench import WORKLOADS, gen_frames, gpu_identity, make_cfg  # noqa: E402


def short_name(name):
    """Kernel name without namespace, template arguments and parameter list."""
    base = name.split("(")[0]
    base = base.split("<")[0]
    return base.split("::")[-1].strip() or name


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--workload", default="fast5", choices=[k for k, v in WORKLOADS.items() if k.startswith("fast")])
    ap.add_argument("--frames", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--trace", default=None, help="keep the chrome trace at this path (default: a temporary file, removed)")
    ap.add_argument("--json", default=None, help="also write the per-kernel table to this file")
    args = ap.parse_args()

    import torch
    from torch.profiler import ProfilerActivity, profile
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
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for i in range(args.warmup, n):
            integ.integrate_depth_device(frames[i][2], d_depth[i].data_ptr(), d_label[i].data_ptr(), w, h, cam.K, ts.cuda_stream)
        integ.sync()
        torch.cuda.synchronize()
    integ.close()

    trace = args.trace or os.path.join(tempfile.mkdtemp(prefix="ksg_trace_"), "trace.json")
    prof.export_chrome_trace(trace)
    with open(trace) as fh:
        events = json.load(fh)["traceEvents"]
    if not args.trace:
        os.remove(trace)
    dev = [e for e in events if e.get("ph") == "X" and e.get("cat") in ("kernel", "gpu_memset", "gpu_memcpy")]
    if not dev:
        raise SystemExit("no device activity in the trace: does this process see the GPU?")
    per = defaultdict(lambda: [0, 0.0])
    for e in dev:
        key = short_name(e["name"]) if e["cat"] == "kernel" else e["name"]
        per[key][0] += 1
        per[key][1] += float(e["dur"])
    busy = sum(float(e["dur"]) for e in dev)
    t0 = min(float(e["ts"]) for e in dev)
    t1 = max(float(e["ts"]) + float(e["dur"]) for e in dev)
    span = t1 - t0
    F = args.frames
    print(f"{args.workload}: {F} traced frames after {args.warmup} warm-up frames; {gpu_identity(0)}")
    print(f"{'launch':34s} {'calls/frame':>11s} {'µs/frame':>9s} {'of span':>8s}")
    rows = sorted(per.items(), key=lambda kv: -kv[1][1])
    for k, (c, d) in rows:
        print(f"{k[:34]:34s} {c / F:11.2f} {d / F:9.1f} {100.0 * d / span:7.1f} %")
    print(f"{'busy (sum of the above)':34s} {'':11s} {busy / F:9.1f} {100.0 * busy / span:7.1f} %")
    print(f"{'span (first start .. last end)':34s} {'':11s} {span / F:9.1f}")
    print(f"{'gaps (span - busy)':34s} {'':11s} {(span - busy) / F:9.1f} {100.0 * (span - busy) / span:7.1f} %")
    if args.json:
        with open(args.json, "w") as fh:
            json.dump({"workload": args.workload, "gpu": gpu_identity(0), "frames": F, "span_us_per_frame": span / F,
                       "busy_us_per_frame": busy / F,
                       "per_launch": {k: {"calls_per_frame": c / F, "us_per_frame": d / F} for k, (c, d) in rows}}, fh, indent=1)


if __name__ == "__main__":
    main()
