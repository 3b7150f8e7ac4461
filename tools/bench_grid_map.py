"""Measures the occupancy grid (gf_grid_map_*) on the GPU and writes profiles/h100_grid_map.json (or --out):
  - keyframe latency (rays, sort, apply; host clock around the synchronous call), with the records (ray steps) per keyframe,
    the longest per-cell run and the updates the exact shortcuts skipped;
  - updatePath rebuild time at 500, 2000 and 5000 keyframes;
  - the same calls on oracle/gm_oracle.c (shared mode, one CPU thread, no shortcut).  The oracle takes every keyframe up to 2000
    and both rebuilds there; the 5000-keyframe rebuild is timed on the oracle over the first 1000 keyframes and scaled by 5, as
    the file says.
Workload: the tool's grid (1500 x 500 cells of 0.05 m, p 0.6 / 0.4 / 0.5), keyframes as the dense map keeps them at 640x480
with DEPTH_DIST 10 and DEPTH_BOUNDARY 10 (2852 samples, depths 0.3 .. 7 m), a forward-looking camera 0.3 m above the body, a
vehicle trajectory wandering over +-30 m.  bel, the image and the occupancy are checked bit for bit against the oracle up to
2000 keyframes; past it each rebuild (same poses) must give back the incremental grid's bel.
Usage: python tools/bench_grid_map.py [--out PATH]"""
import argparse
import json
import math
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from ground_fusion_b200.grid_map import GridMap  # noqa: E402
from oracle.gm_oracle import GridMapOracle  # noqa: E402

W, H, DD, DB = 640, 480, 10, 10
RIC = np.array([[0.0, 0.0, 1.0], [-1.0, 0.0, 0.0], [0.0, -1.0, 0.0]])
TIC = np.array([0.04, 0.03, 0.3])


def keyframe_points(k):
    """2852 camera-frame samples of a 640x480 frame (pinhole 460 / 320 / 240), a floor 0.3 m below the camera and walls, 0.3 .. 7 m."""
    rng = np.random.default_rng(k)
    us, vs = np.meshgrid(np.arange(DB, W - DB, DD), np.arange(DB, H - DB, DD))
    x, y = (us.ravel() - 320.0) / 460.0, (vs.ravel() - 240.0) / 460.0
    d = np.where(y > 0.05, np.minimum(0.3 / np.maximum(y, 1e-3), 7.0), rng.uniform(1.0, 7.0)) + rng.normal(0, 0.01, x.size)
    d = np.clip(d, 0.3, 7.0)
    out = np.zeros((x.size, 6), np.float32)
    out[:, 0], out[:, 1], out[:, 2] = x * d, y * d, d
    out[:, 3:] = 128
    return out


def pose(k):
    t = 0.01 * k
    yaw = 0.9 * t + 0.3 * math.sin(3 * t)
    R = np.array([[math.cos(yaw), -math.sin(yaw), 0], [math.sin(yaw), math.cos(yaw), 0], [0, 0, 1]])
    return R, np.array([30 * math.sin(0.37 * t), 12 * math.sin(0.61 * t), 0.0])


def same(g, o):
    return bool(g.bel().tobytes() == o.bel().tobytes() and g.image().tobytes() == o.image().tobytes()
                and g.occupancy().tobytes() == o.occupancy().tobytes())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_grid_map.json"))
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("no CUDA device: this measurement needs the GPU")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    card = q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(0)
    pts = [keyframe_points(k) for k in range(64)]
    g = GridMap(RIC, TIC, max_points=16 << 20, max_keyframes=6000)
    o = GridMapOracle(RIC, TIC)
    res = {"card": card, "workload": "1500 x 500 grid of 0.05 m; 640x480 keyframes, DEPTH_DIST 10, DEPTH_BOUNDARY 10 (2852 points)",
           "keyframe": [], "rebuild": []}
    Rs, Ps = [], []

    def save():
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)

    ORACLE_UNTIL = 2000
    stats, tg, to = [], [], []
    for k in range(5000):
        R, P = pose(k)
        p = pts[k % len(pts)]
        t0 = time.perf_counter()
        g.addKeyFrame(R, P, p)
        tg.append(time.perf_counter() - t0)
        stats.append(g.stats())
        if k < ORACLE_UNTIL:
            t0 = time.perf_counter()
            o.addKeyFrame(R, P, p)
            to.append(time.perf_counter() - t0)
        Rs.append(R); Ps.append(P)
        n = k + 1
        if n in (100, 500, 2000, 5000):
            recs = [s["records"] for s in stats[1:]]
            entry = {"keyframes": n, "gpu_ms_median": 1e3 * float(np.median(tg[1:])), "gpu_ms_p90": 1e3 * float(np.percentile(tg[1:], 90)),
                     "records_per_keyframe_median": float(np.median(recs)), "records_per_keyframe_max": int(max(recs)),
                     "longest_run": int(max(s["longest_run"] for s in stats)),
                     "applied": int(sum(s["applied"] for s in stats)), "skipped_by_shortcuts": int(sum(s["skipped"] for s in stats))}
            if n <= ORACLE_UNTIL:
                entry["oracle_ms_median"] = 1e3 * float(np.median(to[1:]))
                entry["matches_oracle"] = same(g, o)
            res["keyframe"].append(entry)
            print(entry, flush=True)
            save()
        if n in (500, 2000, 5000):
            before = g.bel().tobytes()
            t = []
            for _ in range(3):                            # the same poses: each rebuild gives back the incremental grid
                t0 = time.perf_counter()
                g.updatePath(np.array(Rs), np.array(Ps))
                t.append(time.perf_counter() - t0)
            st = g.stats()
            entry = {"keyframes": n, "gpu_ms_median": 1e3 * float(np.median(t)), "gpu_ms_all": [1e3 * x for x in t],
                     "records": st["records"], "applied": st["applied"], "skipped_by_shortcuts": st["skipped"], "longest_run": st["longest_run"],
                     "equals_incremental": g.bel().tobytes() == before}
            if n <= ORACLE_UNTIL:
                t0 = time.perf_counter()
                o.updatePath(np.array(Rs), np.array(Ps))
                entry["oracle_ms"] = 1e3 * (time.perf_counter() - t0)
                entry["matches_oracle"] = same(g, o)
            else:
                sub = GridMapOracle(RIC, TIC)
                for j in range(1000):
                    sub.addKeyFrame(Rs[j], Ps[j], pts[j % len(pts)])
                t0 = time.perf_counter()
                sub.updatePath(np.array(Rs[:1000]), np.array(Ps[:1000]))
                entry["oracle_ms"] = 5e3 * (time.perf_counter() - t0)
                entry["oracle_note"] = "the oracle's rebuild over the first 1000 keyframes, times 5"
            res["rebuild"].append(entry)
            print(entry, flush=True)
            save()
    g.close()
    print(json.dumps({"card": card, "keyframe_ms": res["keyframe"][-1]["gpu_ms_median"], "rebuild_ms": [r["gpu_ms_median"] for r in res["rebuild"]]}))


if __name__ == "__main__":
    main()
