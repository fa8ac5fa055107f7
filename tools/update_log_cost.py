"""What the `merged` update log costs and saves, per frame of bench.py's frames (see DESIGN.md §8 and §10).

  python tools/update_log_cost.py [--workloads merged2,merged5] [--frames 12] [--warmup 3] [--capacity 2097152]

Per workload, two integrators fed the same frames, one without and one with the log:
  - frame time from CUDA events around ksg_integrate_depth_device on one stream (log off / on, alternating frame by frame);
  - host wall time of ksg_fetch_update_log against ksg_last_updated_blocks + ksg_export_blocks_by_index of the same frame (what the
    C++ shim's eager sync runs with and without the log; both into host memory, nothing written into layers);
  - log entries and bytes (32 B + 4 C B per entry) against the bytes of the updated blocks, and the frames that overflow --capacity
    (the shim's log size).
Prints one JSON object."""
import argparse
import ctypes as C
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from bench import WORKLOADS, gen_frames, make_cfg  # noqa: E402
from kimera_semantics_b200.capi import Integrator, _ptr  # noqa: E402


def med(x):
    return float(np.median(x)) if len(x) else None


def run(workload, n_frames, warmup, capacity):
    _, w, h, _, Cn, _, _ = WORKLOADS[workload]
    cam, frames = gen_frames(workload, n_frames + warmup)
    off, on = Integrator(make_cfg(workload)), Integrator(make_cfg(workload))
    on.set_update_log(max(capacity, 1 << 23))      # big enough for every frame: the overflow against `capacity` is counted below
    stream = torch.cuda.Stream()
    K = np.asarray(cam.K, np.float32)
    V = 16 ** 3
    res = {"frame_ms_log_off": [], "frame_ms_log_on": [], "fetch_log_ms": [], "fetch_blocks_ms": [], "entries": [], "blocks": []}
    for f, (depth, label, T) in enumerate(frames):
        d_depth = torch.from_numpy(np.ascontiguousarray(depth, np.float32)).cuda()
        d_label = torch.from_numpy(np.ascontiguousarray(label, np.uint8)).cuda()
        torch.cuda.synchronize()
        for name, integ in ((("off", off), ("on", on)) if f % 2 == 0 else (("on", on), ("off", off))):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            with torch.cuda.stream(stream):
                e0.record(stream)
                integ.integrate_depth_device(T, d_depth.data_ptr(), d_label.data_ptr(), w, h, K, stream=stream.cuda_stream)
                e1.record(stream)
            e1.synchronize()
            if f >= warmup:
                res[f"frame_ms_log_{name}"].append(e0.elapsed_time(e1))
        # the same frame's result, fetched both ways from the integrator that keeps the log
        n, hp, pp = C.c_int64(), C.c_void_p(), C.POINTER(C.c_float)()
        t0 = time.perf_counter()
        rc = on.lib.ksg_fetch_update_log(on.handle, C.byref(n), C.byref(hp), C.byref(pp))
        t1 = time.perf_counter()
        assert rc == 0, rc
        nb = int(on.lib.ksg_last_updated_blocks(on.handle, 0, None))
        idx = np.zeros((nb, 3), np.int32)
        found = np.zeros(nb, np.uint8)
        dist, wgt, lab = np.empty((nb, V), np.float32), np.empty((nb, V), np.float32), np.empty((nb, V), np.uint8)
        rgba, srgba, pri = np.empty((nb, V, 4), np.uint8), np.empty((nb, V, 4), np.uint8), np.empty((nb, V, Cn), np.float32)
        t2 = time.perf_counter()
        on.lib.ksg_last_updated_blocks(on.handle, nb, _ptr(idx, C.c_int32))
        rc = on.lib.ksg_export_blocks_by_index(on.handle, nb, _ptr(idx, C.c_int32), _ptr(found, C.c_uint8), _ptr(dist, C.c_float), _ptr(wgt, C.c_float),
                                               _ptr(rgba, C.c_uint8), _ptr(lab, C.c_uint8), _ptr(pri, C.c_float), _ptr(srgba, C.c_uint8))
        t3 = time.perf_counter()
        assert rc == 0, rc
        if f >= warmup:
            res["fetch_log_ms"].append(1e3 * (t1 - t0))
            res["fetch_blocks_ms"].append(1e3 * (t3 - t2))
        res["entries"].append(int(n.value))
        res["blocks"].append(nb)
    off.close()
    on.close()
    entry_bytes = 32 + 4 * Cn
    block_bytes = V * (4 + 4 + 4 + 1 + 4 * Cn + 4)
    return {
        "frames_timed": n_frames,
        "frame_ms_log_off_median": med(res["frame_ms_log_off"]), "frame_ms_log_on_median": med(res["frame_ms_log_on"]),
        "log_pass_ms_median": med(np.array(res["frame_ms_log_on"]) - np.array(res["frame_ms_log_off"])),
        "fetch_log_ms_median": med(res["fetch_log_ms"]), "fetch_blocks_ms_median": med(res["fetch_blocks_ms"]),
        "entries_per_frame": [min(res["entries"]), max(res["entries"])],
        "blocks_per_frame": [min(res["blocks"]), max(res["blocks"])],
        "log_mb_per_frame_max": max(res["entries"]) * entry_bytes / 1e6, "block_mb_per_frame_max": max(res["blocks"]) * block_bytes / 1e6,
        "frames_over_capacity": int(sum(e > capacity for e in res["entries"])), "capacity": capacity,
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="merged2,merged5")
    ap.add_argument("--frames", type=int, default=12)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--capacity", type=int, default=1 << 21)
    a = ap.parse_args()
    out = {"device": torch.cuda.get_device_name(0)}
    for wl in a.workloads.split(","):
        out[wl] = run(wl, a.frames, a.warmup, a.capacity)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
