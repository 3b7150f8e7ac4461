"""Measures the dense colour map (gf_dense_map_*) on the GPU and writes profiles/h100_dense_map.json (or --out):
  - keyframe latency (sampling + insertion + incremental radius filter, host clock around the synchronous call) at cloud sizes of
    about 1e5, 1e6 and 5e6 points;
  - updatePath rebuild time (transform, gate < 5, full filter) at 500, 2000 and 5000 keyframes;
  - the same calls on oracle/dm_oracle.c, one CPU thread: a sequential restatement of the reference's semantics, not PCL.
Workload: 640x480 keyframes sampled every 10th pixel (DEPTH_DIST 10, DEPTH_BOUNDARY 10: 2852 samples), depths 0.1 .. 2.3 m, a
trajectory that keeps reaching new ground so the cloud grows by ~2.5k points per keyframe, as a long mapping run does.  The GPU
map's cloud, keyframe lists and filter are checked bit for bit against the oracle at every measured point.
Usage: python tools/bench_dense_map.py [--out PATH]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from ground_fusion_b200.dense_map import DenseMap  # noqa: E402
from ground_fusion_b200.synth import idc_params8  # noqa: E402
from oracle.dm_oracle import DenseMapOracle  # noqa: E402

W, H = 640, 480


def frames(n=8, seed=0):
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(n):
        ys, xs = np.mgrid[0:H, 0:W]
        d = 400 + 1900 * (0.5 * xs / W + 0.5 * ys / H) + rng.normal(0, 30, (H, W))
        d[rng.random((H, W)) < 0.05] = 0
        out.append((rng.integers(0, 256, (H, W, 3)).astype(np.uint8), np.clip(d, 0, 65535).astype(np.uint16)))
    return out


def pose(k):
    a = 0.002 * k
    R = np.array([[np.cos(a), -np.sin(a), 0], [np.sin(a), np.cos(a), 0], [0, 0, 1]])
    return R, np.array([0.25 * k * np.cos(0.3 * a), 0.25 * k * np.sin(0.3 * a) + 0.1 * np.sin(0.05 * k), -0.4])


def same(g, o):
    gx, gr = g.cloud()
    ox, orr = o.cloud()
    return bool(gx.tobytes() == ox.tobytes() and np.array_equal(gr, orr) and np.array_equal(g.filtered()[2], o.filtered()[2]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_dense_map.json"))
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("no CUDA device: this measurement needs the GPU")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    card = q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(0)
    fr = frames()
    g = DenseMap(W, H, idc_params8(), 10, 10, max_points=16 << 20, max_keyframes=6000)
    o = DenseMapOracle(W, H, idc_params8(), 10, 10, np.eye(3), np.zeros(3))
    Rs, Ps = [], []
    k = 0

    def save():                                           # after every record: a cut-short run keeps what it measured
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)

    def add(timed):
        nonlocal k
        R, P = pose(k)
        rgb, depth = fr[k % len(fr)]
        t0 = time.perf_counter()
        g.addKeyFrame(R, P, rgb, depth)
        tg = time.perf_counter() - t0
        t0 = time.perf_counter()
        o.addKeyFrame(R, P, rgb, depth, filter=timed)
        to = time.perf_counter() - t0
        Rs.append(R); Ps.append(P)
        k += 1
        return tg, to

    add(False)                                            # module load, first launches
    res = {"card": card, "workload": "640x480 keyframes, DEPTH_DIST 10, DEPTH_BOUNDARY 10 (2852 samples), IDC camera with distortion",
           "keyframe": [], "rebuild": []}
    size_targets = [100_000, 1_000_000, 5_000_000]
    kf_targets = [500, 2000, 5000]
    while size_targets or kf_targets:
        if size_targets and g.size()[0] >= size_targets[0]:
            tg, to = [], []
            for i in range(5):
                a, b = add(i == 4)                        # the oracle filters (a full recount, timed) on the last only
                tg.append(a)
                if i == 4:
                    to.append(b)
            res["keyframe"].append({"cloud_points": g.size()[0], "gpu_ms_median": 1e3 * float(np.median(tg)), "gpu_ms_all": [1e3 * t for t in tg],
                                    "oracle_restatement_ms": 1e3 * to[0], "matches_oracle": same(g, o)})
            print(res["keyframe"][-1], flush=True)
            save()
            size_targets.pop(0)
            continue
        if kf_targets and len(Rs) >= kf_targets[0]:
            tg = []
            for _ in range(3):                            # the same poses: each rebuild yields the same map
                t0 = time.perf_counter()
                g.updatePath(np.array(Rs), np.array(Ps))
                tg.append(time.perf_counter() - t0)
            t0 = time.perf_counter()
            o.updatePath(np.array(Rs), np.array(Ps))
            to = time.perf_counter() - t0
            res["rebuild"].append({"keyframes": len(Rs), "cloud_points": g.size()[0], "gpu_ms_median": 1e3 * float(np.median(tg)),
                                   "gpu_ms_all": [1e3 * t for t in tg], "oracle_restatement_ms": 1e3 * to, "matches_oracle": same(g, o)})
            print(res["rebuild"][-1], flush=True)
            save()
            kf_targets.pop(0)
            continue
        add(False)
    g.close()
    print(json.dumps({"card": card, "keyframe_ms": [r["gpu_ms_median"] for r in res["keyframe"]],
                      "rebuild_ms": [r["gpu_ms_median"] for r in res["rebuild"]]}))


if __name__ == "__main__":
    main()
