"""Round time of adding one keyframe to each of K dense maps (and K occupancy grids) on the GPU: one group call
(DenseMapGroup / GridMapGroup), K sequential single calls from one thread, and K host threads with one map each.

640 x 480 keyframes, DEPTH_DIST = DEPTH_BOUNDARY = 10 as in bench_dense_map.py; K in {1, 2, 4, 8, 16, 32}; two cloud sizes per
member, about 1e5 and 1e6 points (each member's cloud is grown by group calls with keyframes shifted to fresh voxels).  The grids
are the tool's 1500 x 500, fed each member's last dense keyframe (host points); their cost does not depend on the cloud.  Times
are host clock per round ending in a device synchronise (median of --rounds); the group's kernel time is the sum of the CUDA
kernels torch.profiler records over --rounds group rounds.  One JSON line per (stage, K) and a summary line with the card's
name and power limit.
    python tools/bench_map_group.py [--rounds 5] [--out profiles/h100_map_group.json]"""
import argparse
import json
import os
import subprocess
import sys
import threading
import time

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))


def _card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        name, pl = [x.strip() for x in q.stdout.strip().splitlines()[0].split(",")]
        return name, pl
    except Exception as e:                                # noqa: BLE001
        return "unknown (%s)" % e, "unknown"


def _kernel_ms(fn, rounds):
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(rounds):
            fn()
        torch.cuda.synchronize()
    tot = 0.0
    for e in prof.key_averages():
        t = getattr(e, "self_device_time_total", None)
        tot += (t if t is not None else e.self_cuda_time_total)
    return tot / 1000.0 / rounds


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--ks", default="1,2,4,8,16,32")
    ap.add_argument("--sizes", default="100000,1000000")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    from ground_fusion_b200.dense_map import DenseMap, DenseMapGroup
    from ground_fusion_b200.grid_map import GridMap, GridMapGroup
    from ground_fusion_b200.synth import SyntheticStream, idc_params8
    if not torch.cuda.is_available():
        sys.exit("no CUDA device: this benchmark measures the GPU")
    ks = [int(v) for v in a.ks.split(",")]
    Kmax = max(ks)
    name, pl = _card()
    st = SyntheticStream(seed=0, plane_dist=2.0)
    frames = []
    for k in range(8):
        R, C = st.pose(3 * k)
        frames.append((R.T, C, st.color(3 * k), st.frame(3 * k)[2]))
    maps = [DenseMap(640, 480, idc_params8(), 10, 10, max_points=1 << 21, max_keyframes=4096) for _ in range(Kmax)]
    grids = [GridMap(max_records=1 << 22) for _ in range(Kmax)]
    fill = DenseMapGroup(maps)
    rnd = [0]                                         # rounds so far: round r's keyframes sit 4 r m along x, in fresh voxels

    def frame(i, r):
        R, C, rgb, depth = frames[(r + i) % len(frames)]
        return R, C + np.array([4.0 * r, 0.0, 0.0]), rgb, depth

    def grow(target):
        while min(m.size()[0] for m in maps) < target:
            rnd[0] += 1
            fs = [frame(i, rnd[0]) for i in range(Kmax)]
            _, status = fill.addKeyFrames(range(Kmax), [f[0] for f in fs], [f[1] for f in fs], [f[2] for f in fs], [f[3] for f in fs])
            if status.any():
                sys.exit("filling failed: %s" % status)

    lines = []
    for target in [int(v) for v in a.sizes.split(",")]:
        grow(target)
        pts = [m.keyframePoints(m.size()[2] - 1) for m in maps]
        for K in ks:
            dg, gg = DenseMapGroup(maps[:K]), GridMapGroup(grids[:K])

            def d_group():
                rnd[0] += 1
                fs = [frame(i, rnd[0]) for i in range(K)]
                dg.addKeyFrames(range(K), [f[0] for f in fs], [f[1] for f in fs], [f[2] for f in fs], [f[3] for f in fs])
                dg.members[0].size()                      # the members' reads follow the group's work

            def d_seq():
                rnd[0] += 1
                for i in range(K):
                    maps[i].addKeyFrame(*frame(i, rnd[0]))

            def d_thr():
                rnd[0] += 1
                ts = [threading.Thread(target=lambda i=i, r=rnd[0]: maps[i].addKeyFrame(*frame(i, r))) for i in range(K)]
                for t in ts:
                    t.start()
                for t in ts:
                    t.join()

            def g_group():
                gg.addKeyFrames(range(K), [f[0] for f in frames[:1] * K], [f[1] for f in frames[:1] * K], pts[:K])

            def g_seq():
                for i in range(K):
                    grids[i].addKeyFrame(frames[0][0], frames[0][1], pts[i])

            def g_thr():
                ts = [threading.Thread(target=lambda i=i: grids[i].addKeyFrame(frames[0][0], frames[0][1], pts[i])) for i in range(K)]
                for t in ts:
                    t.start()
                for t in ts:
                    t.join()

            res = {}
            for label, fn in (("dense_group", d_group), ("dense_sequential", d_seq), ("dense_threads", d_thr),
                              ("grid_group", g_group), ("grid_sequential", g_seq), ("grid_threads", g_thr)):
                fn()                                      # warm-up
                torch.cuda.synchronize()
                ts = []
                for _ in range(a.rounds):
                    t0 = time.perf_counter()
                    fn()
                    torch.cuda.synchronize()
                    ts.append((time.perf_counter() - t0) * 1e3)
                res[label + "_ms"] = round(float(np.median(ts)), 3)
            res["dense_group_kernel_ms"] = round(_kernel_ms(d_group, a.rounds), 3)
            res["grid_group_kernel_ms"] = round(_kernel_ms(g_group, a.rounds), 3)
            line = dict(stage="cloud~%g" % target, K=K, cloud_per_member=int(np.mean([m.size()[0] for m in maps[:K]])), **res)
            print(json.dumps(line), flush=True)
            lines.append(line)
            dg.close(); gg.close()
    summary = dict(bench="map_group", gpu=name, power_limit=pl, rounds=a.rounds, frame="640x480", depth_dist=10, depth_boundary=10,
                   grid="1500x500", results=lines)
    print(json.dumps(dict(bench="map_group", gpu=name, power_limit=pl)))
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(summary, f, indent=1)
    fill.close()
    for x in maps + grids:
        x.close()


if __name__ == "__main__":
    main()
