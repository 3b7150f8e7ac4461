"""Cost of the front end's `equalize` option (CLAHE, clip 40, 8x8 tiles, on every frame) on the C2 workload.

Prints one JSON line: frames/s with and without the option, one stream and eight streams (one host thread,
gf_tracker_track_batch_multi), plain and equalised runs alternating in one process on the same frames, measured the way
bench.py measures its headline (100-frame steps, frames resident in HBM = value, pinned host frames = e2e); and the CPU arm
with cv2.createCLAHE().apply in front of the reference's OpenCV calls and glue.

    python tools/bench_equalize.py [--rounds 2] [--steps 20] [--warmup 3]
"""
import argparse
import contextlib
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402

import bench  # noqa: E402


class EqualizingStream(bench.Stream):
    """bench.Stream whose tracker equalises every frame (gf_tracker_set_equalize before its first frame)."""

    def __init__(self, *a, **k):
        super().__init__(*a, **k)
        self.tr.set_equalize(40.0, (8, 8))


@contextlib.contextmanager
def equalized(on):
    """bench.fe_line builds its trackers through bench.Stream: swap in the equalising one for the duration."""
    plain = bench.Stream
    if on:
        bench.Stream = EqualizingStream
    try:
        yield
    finally:
        bench.Stream = plain


def cpu_arm(gray, depth, wl, frames, warm=20):
    """frames/s of the reference's CPU path with `equalize` set: cv2.createCLAHE().apply, then its three OpenCV calls + glue."""
    import cv2
    from oracle.fe_oracle import IDC_CAM, FeatureTrackerOracleFast, PinholeCamera
    cam = PinholeCamera(**IDC_CAM)
    ft = FeatureTrackerOracleFast(cam, wl["max_cnt"], wl["min_dist"], 1, 1)
    clahe = cv2.createCLAHE()
    n = len(gray)
    t_clahe = 0.0
    for k in range(warm + frames):
        if k == warm:
            t0, ft.t_cv, t_clahe = time.perf_counter(), 0.0, 0.0
        g = gray[bench.tri(k, n)]
        t1 = time.perf_counter()
        g = clahe.apply(g)
        t_clahe += time.perf_counter() - t1
        ft.trackImage(k / 30.0, g, depth[bench.tri(k, n)])
    dt = time.perf_counter() - t0
    return {"value": frames / dt, "clahe_ms_per_frame": 1e3 * t_clahe / frames, "opencv_calls_only": frames / (ft.t_cv + t_clahe),
            "frames": frames, "threads": cv2.getNumThreads()}


def gpu_name_and_power_limit():
    try:
        q = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], text=True)
        return q.strip()
    except Exception:
        return torch.cuda.get_device_name(0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--cpu-frames", type=int, default=100)
    args = ap.parse_args()
    wl = bench.WORKLOADS["C2"]
    ring = bench.Ring(0, wl, torch)

    def barrier():
        torch.cuda.synchronize()

    runs = {k: [] for k in ("plain_1", "equalize_1", "plain_8", "equalize_8")}
    for _ in range(args.rounds):
        for on in (False, True):
            name = "equalize" if on else "plain"
            with equalized(on):
                r1 = bench.fe_line(wl, [ring], 0, 1, args.steps, args.warmup, barrier, None, lambda v: v)
                r8 = bench.fe_line(wl, [ring], 0, 8, max(4, args.steps // 2), 2, barrier, None, lambda v: v)
            runs[name + "_1"].append({"value": r1["value"], "e2e": r1["e2e"], "gpu_launches_per_frame": r1["gpu_launches"] / (args.steps * bench.FRAMES_PER_STEP)})
            runs[name + "_8"].append({"value": r8["value"], "e2e": r8["e2e"]})
    med = {k: {"value": float(np.median([r["value"] for r in v])), "e2e": float(np.median([r["e2e"] for r in v]))} for k, v in runs.items()}
    cpu = cpu_arm(ring.gray[:60], ring.depth[:60], wl, args.cpu_frames)
    out = {"metric": "tracker_frames_per_sec", "unit": "frames/s", "workload": wl["name"] + "; equalize: cv::createCLAHE() (clip 40, 8x8 tiles) on every frame",
           "gpu": gpu_name_and_power_limit(), "rounds": args.rounds, "steps": args.steps, "warmup": args.warmup,
           "median": med, "runs": runs,
           "equalize_vs_plain": {"streams_1": med["equalize_1"]["value"] / med["plain_1"]["value"], "streams_8": med["equalize_8"]["value"] / med["plain_8"]["value"]},
           "cpu_equalize": cpu, "speedup_vs_cpu": med["equalize_1"]["value"] / cpu["value"]}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
