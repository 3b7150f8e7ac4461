"""Tracker groups (gf_tracker_group) against independent streams (gf_tracker_track_batch_multi) on the C2 workload of bench.py.

K trackers of the C2 configuration share one ring of distinct 640x480 RGB-D frames (larger than L2; member i starts 17 i frames
further on), 100-frame steps.  At each K the same trackers run TrackerGroup.trackBatch and FeatureTracker.trackBatchMulti
alternately in one process, frames resident in HBM (value) and in pinned host memory (e2e), for --rounds rounds; the JSON line
gives medians and ranges in frames/s summed over the K cameras, and the device time of one step (CUDA events from its first copy
to its result copy: the latency each camera sees, which for a lockstep group ends with its slowest member).  Also in the same run:
  host_us_per_frame: host time inside the submit calls, K = 8, frames in HBM (a host clock around each call, ctypes included;
      ctypes_call_us is the cost of an empty call for comparison), for gf_tracker_submit of a device frame as gf_tracker_track_batch_multi
      issues it and for gf_tracker_group_submit divided by K;
  kernels_k8: per-kernel device times of one K = 8 run of each path (torch.profiler);
  gpu: the card's name and power limit.

    python tools/bench_fe_group.py [--rounds 3] [--steps 10] [--warmup 2] [--ks 1,2,4,8,16,32] [--out FILE]
"""
import argparse
import ctypes
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402

import bench  # noqa: E402
from bench_equalize import gpu_name_and_power_limit  # noqa: E402
from ground_fusion_b200 import _lib  # noqa: E402
from ground_fusion_b200.feature_tracker import FeatureTracker, TrackerGroup  # noqa: E402
from ground_fusion_b200.synth import idc_params8  # noqa: E402

N = bench.FRAMES_PER_STEP


class Rig:
    """K trackers on the shared ring, and the group of the same trackers."""

    def __init__(self, ring, wl, K):
        self.ring, self.K = ring, K
        self.tr = [FeatureTracker(wl["w"], wl["h"], idc_params8(), wl["max_cnt"], wl["min_dist"], 1, 1) for _ in range(K)]
        self.group = TrackerGroup(self.tr)
        self.k = [17 * i for i in range(K)]

    def batch(self, n):
        times, idx = [], []
        for i in range(self.K):
            idx.append([bench.tri(self.k[i] + j, self.ring.n) for j in range(n)])
            times.append([(self.k[i] + j) / 30.0 for j in range(n)])
            self.k[i] += n
        return times, idx

    def run(self, path, mode, steps, n=N):
        g, d = self.ring.ptr[mode]
        lat = []
        for _ in range(steps):
            times, idx = self.batch(n)
            gp, dp = [[g[j] for j in row] for row in idx], [[d[j] for j in row] for row in idx]
            if path == "group":
                self.group.trackBatch(times, gp, dp, on_device=(mode == "device"), want=False)
            else:
                FeatureTracker.trackBatchMulti(self.tr, times, gp, dp, on_device=(mode == "device"), want=False)
            lat.append(self.tr[0].last_device_ms())
        return lat

    def close(self):
        self.group.close()
        for t in self.tr:
            t.close()


def timed(rig, path, mode, steps, warmup):
    rig.run(path, mode, warmup)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    lat = rig.run(path, mode, steps)
    torch.cuda.synchronize()
    return rig.K * steps * N / (time.perf_counter() - t0), float(np.median(lat))


def host_cost(ring, wl, K=8, frames=400):
    """Host microseconds per frame spent inside the submit calls, frames in HBM."""
    L = _lib.lib()
    g, d = ring.ptr["device"]
    rig = Rig(ring, wl, K)
    rig.run("multi", "device", 1, 20)
    rig.run("group", "device", 1, 20)
    ns_multi, ns_group = 0, 0
    for k in range(frames):                 # the submit / wait order of gf_tracker_track_batch_multi
        for i, t in enumerate(rig.tr):
            j = bench.tri(rig.k[i] + k, ring.n)
            t0 = time.perf_counter_ns()
            _lib.check(L.gf_tracker_submit(t._h, (rig.k[i] + k) / 30.0, g[j], 0, d[j], 0, 1, None, 0))
            ns_multi += time.perf_counter_ns() - t0
        if k >= 1:
            for t in rig.tr:
                t.wait()
    for t in rig.tr:
        t.wait()
    rig.k = [x + frames for x in rig.k]
    times = (ctypes.c_double * K)()
    gp, dp = (ctypes.c_void_p * K)(), (ctypes.c_void_p * K)()
    for k in range(frames):
        for i in range(K):
            j = bench.tri(rig.k[i] + k, ring.n)
            times[i], gp[i], dp[i] = (rig.k[i] + k) / 30.0, g[j], d[j]
        t0 = time.perf_counter_ns()
        _lib.check(L.gf_tracker_group_submit(rig.group._h, times, gp, 640, dp, 1280, 1, None, None))
        ns_group += time.perf_counter_ns() - t0
        if k >= 1:
            rig.group.wait()
    rig.group.wait()
    t0 = time.perf_counter_ns()
    for _ in range(10000):
        L.gf_kernel_launch_count()
    empty = (time.perf_counter_ns() - t0) / 10000
    rig.close()
    return {"K": K, "frames": frames, "track_batch_multi_submit_us": ns_multi / 1e3 / (K * frames),
            "group_submit_us_per_member": ns_group / 1e3 / (K * frames), "group_submit_us_per_step": ns_group / 1e3 / frames,
            "ctypes_call_us": empty / 1e3}


def kernels(ring, wl, K=8):
    """Per-kernel device time of one 100-frame step per path (torch.profiler, CUDA activity)."""
    from torch.profiler import ProfilerActivity, profile
    rig = Rig(ring, wl, K)
    out = {}
    for path in ("multi", "group"):
        rig.run(path, "device", 1)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            rig.run(path, "device", 1)
            torch.cuda.synchronize()
        rows = {}
        for e in prof.key_averages():
            if e.device_type.name == "CUDA" and e.count > 0:
                us = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0.0)
                rows[e.key] = {"calls": int(e.count), "total_us": float(us), "mean_us": float(us) / e.count}
        out[path] = dict(sorted(rows.items(), key=lambda kv: -kv[1]["total_us"])[:24])
    rig.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--ks", default="1,2,4,8,16,32")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    wl = bench.WORKLOADS["C2"]
    ring = bench.Ring(0, wl, torch)
    ks = [int(x) for x in args.ks.split(",")]
    res = {K: {p: {m: [] for m in ("value", "e2e", "latency_ms")} for p in ("group", "multi")} for K in ks}
    for _ in range(args.rounds):
        for K in ks:
            rig = Rig(ring, wl, K)
            for path in ("multi", "group"):
                v, lat = timed(rig, path, "device", args.steps, args.warmup)
                e, _ = timed(rig, path, "host", args.steps, 1)
                r = res[K][path]
                r["value"].append(v); r["e2e"].append(e); r["latency_ms"].append(lat)
            rig.close()
    summary = {}
    for K in ks:
        summary[K] = {}
        for p in ("group", "multi"):
            summary[K][p] = {m: {"median": float(np.median(v)), "min": float(np.min(v)), "max": float(np.max(v))} for m, v in res[K][p].items()}
        summary[K]["group_vs_multi_value"] = summary[K]["group"]["value"]["median"] / summary[K]["multi"]["value"]["median"]
        summary[K]["group_vs_multi_e2e"] = summary[K]["group"]["e2e"]["median"] / summary[K]["multi"]["e2e"]["median"]
    out = {"metric": "tracker_frames_per_sec_all_cameras", "unit": "frames/s", "workload": wl["name"] + "; K cameras, 100-frame steps",
           "gpu": gpu_name_and_power_limit(), "rounds": args.rounds, "steps": args.steps, "warmup": args.warmup,
           "note": "value: frames in HBM; e2e: pinned host frames; latency_ms: device time of one step (last step of a batch), "
                   "first copy to result copy; group = TrackerGroup.trackBatch, multi = FeatureTracker.trackBatchMulti on the same trackers",
           "by_k": summary, "host_us_per_frame": host_cost(ring, wl), "kernels_k8": kernels(ring, wl)}
    line = json.dumps(out)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
