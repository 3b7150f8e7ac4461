"""Cost of trackImagebox (`use_yolo`) on the C2 workload: 8 moving boxes on every frame against plain trackImage.

Prints one JSON line: frames/s with and without boxes, one stream and eight streams (one host thread,
gf_tracker_track_batch_multi), plain and boxed runs alternating in one process on the same frames, measured the way bench.py
measures its headline (100-frame steps, frames resident in HBM = value, pinned host frames = e2e), with the card's name and
power limit read in the same run.  The boxes go in through the `boxes=` argument of trackBatch / trackBatchMulti, so the time
includes building the per-frame box lists in Python.  `finalize_us` isolates the device: the k_select_finalize stage (CUDA
events, profiling mode, one frame at a time) with and without the boxes, medians over the same frames.

    python tools/bench_boxes.py [--rounds 3] [--steps 20] [--warmup 3]
"""
import argparse
import contextlib
import json
import math
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402

import bench  # noqa: E402
from bench_equalize import gpu_name_and_power_limit  # noqa: E402
from ground_fusion_b200.feature_tracker import FeatureTracker  # noqa: E402

N_BOXES = 8
_cache = {}


def boxes_at(t, w=640, h=480):
    """8 boxes of 60-160 px on their own circular paths through the image at frame time t (int64 corners, as darknet_ros's)."""
    k = int(round(t * 30.0))
    if k not in _cache:
        out = []
        for i in range(N_BOXES):
            a = 0.05 * k * (1 + 0.3 * i) + i
            cx, cy = w / 2 + 0.35 * w * math.cos(a), h / 2 + 0.35 * h * math.sin(1.3 * a)
            bw, bh = 60 + 12 * i, 50 + 10 * i
            out.append([int(cx - bw / 2), int(cy - bh / 2), int(cx + bw / 2), int(cy + bh / 2)])
        _cache[k] = np.array(out, np.int64)
    return _cache[k]


@contextlib.contextmanager
def boxed(on):
    """bench's loops call trackBatch / trackBatchMulti without boxes: for the duration, give every frame its boxes."""
    plain_batch, plain_multi = FeatureTracker.trackBatch, FeatureTracker.trackBatchMulti
    if on:
        def batch(self, times, *a, **k):
            k["boxes"] = [boxes_at(t) for t in times]
            return plain_batch(self, times, *a, **k)

        def multi(trackers, times, *a, **k):
            k["boxes"] = [[boxes_at(t) for t in row] for row in times]
            return plain_multi(trackers, times, *a, **k)
        FeatureTracker.trackBatch, FeatureTracker.trackBatchMulti = batch, staticmethod(multi)
    try:
        yield
    finally:
        FeatureTracker.trackBatch, FeatureTracker.trackBatchMulti = plain_batch, staticmethod(plain_multi)


def finalize_stage_us(ring, wl, frames=300):
    """Median k_select_finalize time (us) of plain trackImage and of trackImagebox with the 8 boxes, frames alternating."""
    sc = wl["w"] / 640.0
    from ground_fusion_b200.synth import idc_params8
    p8 = idc_params8()
    p8 = [p8[0] * sc, p8[1] * sc, p8[2] * sc, p8[3] * sc] + p8[4:]
    trs = [FeatureTracker(wl["w"], wl["h"], p8, wl["max_cnt"], wl["min_dist"], 1, 1) for _ in range(2)]
    for tr in trs:
        tr.set_profiling(True)
    ms = {False: [], True: []}
    for k in range(frames):
        g, d = ring.gray[bench.tri(k, ring.n)], ring.depth[bench.tri(k, ring.n)]
        trs[0].trackImageRaw(k / 30.0, g, d)
        trs[1].trackImageboxRaw(k / 30.0, boxes_at(k / 30.0), g, d)
        if k >= 20:
            for on, tr in zip((False, True), trs):
                ms[on].append(tr.last_stage_ms()["finalize"])
    for tr in trs:
        tr.close()
    return {"plain": 1e3 * float(np.median(ms[False])), "boxes": 1e3 * float(np.median(ms[True])), "frames": frames - 20}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    wl = bench.WORKLOADS["C2"]
    ring = bench.Ring(0, wl, torch)

    def barrier():
        torch.cuda.synchronize()

    runs = {k: [] for k in ("plain_1", "boxes_1", "plain_8", "boxes_8")}
    for _ in range(args.rounds):
        for on in (False, True):
            name = "boxes" if on else "plain"
            with boxed(on):
                r1 = bench.fe_line(wl, [ring], 0, 1, args.steps, args.warmup, barrier, None, lambda v: v)
                r8 = bench.fe_line(wl, [ring], 0, 8, max(4, args.steps // 2), 2, barrier, None, lambda v: v)
            runs[name + "_1"].append({"value": r1["value"], "e2e": r1["e2e"], "gpu_launches_per_frame": r1["gpu_launches"] / (args.steps * bench.FRAMES_PER_STEP)})
            runs[name + "_8"].append({"value": r8["value"], "e2e": r8["e2e"]})
    med = {k: {"value": float(np.median([r["value"] for r in v])), "e2e": float(np.median([r["e2e"] for r in v]))} for k, v in runs.items()}
    fin = finalize_stage_us(ring, wl)
    out = {"metric": "tracker_frames_per_sec", "unit": "frames/s",
           "workload": wl["name"] + "; boxes: trackImagebox with %d moving boxes on every frame" % N_BOXES,
           "gpu": gpu_name_and_power_limit(), "rounds": args.rounds, "steps": args.steps, "warmup": args.warmup,
           "median": med, "runs": runs,
           "boxes_vs_plain": {"streams_1": med["boxes_1"]["value"] / med["plain_1"]["value"], "streams_8": med["boxes_8"]["value"] / med["plain_8"]["value"],
                              "streams_1_e2e": med["boxes_1"]["e2e"] / med["plain_1"]["e2e"], "streams_8_e2e": med["boxes_8"]["e2e"] / med["plain_8"]["e2e"]},
           "finalize_us": fin}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
