"""Host time per frame of the FeatureManager stage: feature_manager.FeatureManager (lists in Python, one stateless gf_fm_* call
per loop) against feature_window.FeatureWindow (the table resident on the GPU, gf_fm_window).

The stage is what one processImage does around the solve: addFeatureCheckParallax, triangulate, the factor loop (Python rows
+ set_visual against fillProblem), setDepth, movingConsistencyCheckW + removeOutlier, predictPtsInNextFrame, the window slide's
removal and removeFailures.  The solve itself is left out: setDepth gets the depth vector back unchanged.  Two streams:
  c2   the frames the tracker produces on the 64-frame synthetic replay stream (150 features per frame)
  c3   a synthetic table with 300 features per frame and track lengths as on c2
Both arms run in one process, alternating, `--rounds` times; medians and ranges are reported, and the device time of every
FeatureWindow operation from CUDA events.  The same stage is also timed from C++ alone, so that Python's share is visible:
`adaptor/harness fm-bench` keeps the list in a std::list and calls the stateless gf_fm_* entry points, against gf_fm_window_*
("c_abi" in the result).  Needs a GPU: there is no CPU fallback.

    python tools/bench_fm_window.py --out profiles/h100_fm_window.json
"""
import argparse
import json
import os
import struct
import subprocess
import sys
import tempfile
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from ground_fusion_b200.ba_problem import Problem                    # noqa: E402
from ground_fusion_b200.feature_manager import FeatureManager        # noqa: E402
from ground_fusion_b200.feature_window import FeatureWindow          # noqa: E402


def poses():
    Ps = np.array([[0.12 * k, 0.03 * np.sin(0.5 * k), 0.02 * k] for k in range(11)])
    Rs = np.array([[[np.cos(0.02 * k), 0, np.sin(0.02 * k)], [0, 1, 0], [-np.sin(0.02 * k), 0, np.cos(0.02 * k)]] for k in range(11)])
    return Ps, Rs, np.zeros(3), np.eye(3)


def c2_frames(n):
    from ground_fusion_b200.feature_tracker import FeatureTracker
    from ground_fusion_b200.synth import IDC_CAM, SyntheticStream
    cam = dict(IDC_CAM, k1=0.0, k2=0.0, p1=0.0, p2=0.0)
    tr = FeatureTracker(640, 480, [cam[k] for k in ("fx", "fy", "cx", "cy", "k1", "k2", "p1", "p2")], 150, 30, 1, 1)
    st = SyntheticStream(seed=0)
    out = [tr.trackImage(*st.frame(k)) for k in range(n)]
    tr.close()
    return out


def c3_frames(n, per_frame=300, seed=0):
    """per_frame ids per frame; each frame a tenth of them is replaced by new ids, the rest move a little."""
    rng = np.random.default_rng(seed)
    live = {i: np.array([rng.uniform(-0.5, 0.5), rng.uniform(-0.4, 0.4), 1, 0, 0, 0, 0, rng.uniform(1.0, 3.5)]) for i in range(per_frame)}
    nxt, out = per_frame, []
    for _ in range(n):
        out.append({k: v.copy() for k, v in live.items()})
        for k in list(live)[::10]:
            del live[k]
            live[nxt] = np.array([rng.uniform(-0.5, 0.5), rng.uniform(-0.4, 0.4), 1, 0, 0, 0, 0, rng.uniform(1.0, 3.5)]); nxt += 1
        for v in live.values():
            v[0] += 0.004; v[1] += 0.001
    return out


def python_factor_loop(fm):
    feats = list(fm.iter_ba_features())
    pb = Problem(11, len(feats))
    rows = []
    for k, (start, obs, est_depth, flag) in enumerate(feats):
        pb.para_feature[k] = 1.0 / est_depth
        pb.feature_const[k] = 1 if flag == 1 else 0
        p0, v0, t0 = obs[0]
        for a in range(1, len(obs)):
            pj, vj, tj = obs[a]
            rows.append((start, start + a, k, p0, pj, v0, vj, t0, tj))
    pb.set_visual(rows)
    return pb, len(feats)


def c_abi(frames, P, rounds):
    """The stage through the C ABI alone (adaptor/harness fm-bench): {arm: {stage_us, factor_loop_us}}."""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    with tempfile.TemporaryDirectory() as tmp:
        subprocess.check_call(["make", "-s", "-C", os.path.join(root, "adaptor")])
        Ps, Rs, tic, ric = P
        with open(os.path.join(tmp, "in.bin"), "wb") as f:
            f.write(struct.pack("<2i2d33d99d3d9d", rounds, len(frames), 10.0 / 600.0, 4.0, *Ps.ravel(), *Rs.ravel(), *tic, *ric.ravel()))
            for fr in frames:
                f.write(struct.pack("<i", len(fr)) + b"".join(struct.pack("<i8d", k, *fr[k][:8]) for k in sorted(fr)))
        subprocess.check_call([os.path.join(root, "adaptor", "_build", "harness"), "fm-bench", os.path.join(tmp, "in.bin"), os.path.join(tmp, "out.json")])
        return json.load(open(os.path.join(tmp, "out.json")))


def run(fm, frames, P, device_ms=None):
    """One pass of the stream; returns (seconds per steady-state frame, seconds per factor loop, factors per loop)."""
    Ps, Rs, tic, ric = P
    on_device = isinstance(fm, FeatureWindow)
    t_frame, t_fill, n_rows = [], [], []

    def op(name, f, *a):
        r = f(*a)
        if device_ms is not None:
            device_ms.setdefault(name, []).append(fm.last_device_ms())
        return r

    for k, image in enumerate(frames):
        fc = min(k, 10)
        t0 = time.perf_counter()
        margin_old = op("add_frame", fm.addFeatureCheckParallax, fc, image, 0.0)
        if fc == 10:
            op("triangulate", fm.triangulateAll, fc, Ps, Rs, tic, ric)
            t1 = time.perf_counter()
            if on_device:
                pb = Problem(11, 0); n = op("fill_problem", fm.fillProblem, pb)
            else:
                pb, n = python_factor_loop(fm)
            t_fill.append(time.perf_counter() - t1); n_rows.append(pb.n_visual)
            op("set_depth", fm.setDepth, pb.para_feature[:n])
            # the poses are not the stream's, so the check flags most landmarks: only a few of them go, as on a real window
            op("remove_ids", fm.removeOutlier, set(sorted(op("outliers", fm.movingConsistencyCheckW, Ps, Rs, tic, ric))[:3]))
            op("predict_next", fm.predictPtsInNextFrame, fc, Ps, Rs, tic, ric)
            if margin_old or k % 3 == 0:
                op("remove_back_shift_depth", fm.removeBackShiftDepth, Rs[0], Ps[0], Rs[1], Ps[1])
            else:
                op("remove_front", fm.removeFront, fc)
            op("remove_failures", fm.removeFailures)
            if on_device:
                fm.size()                     # the frame's work has finished on the device before the clock stops
            t_frame.append(time.perf_counter() - t0)
    return float(np.median(t_frame)), float(np.median(t_fill)), float(np.median(n_rows))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=64)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_fm_window needs a GPU")
    card = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"]).decode().strip()
    P = poses()
    res = {"card": card, "frames": a.frames, "rounds": a.rounds, "unit": "microseconds of host time per frame, median over the frames of a pass"}
    for name, frames in (("c2", c2_frames(a.frames)), ("c3", c3_frames(a.frames))):
        run(FeatureManager(depth_threshold=4.0), frames, P); w = FeatureWindow(depth_threshold=4.0); run(w, frames, P); w.close()       # warm-up
        arms = {"FeatureManager": [], "FeatureWindow": []}
        for _ in range(a.rounds):
            arms["FeatureManager"].append(run(FeatureManager(depth_threshold=4.0), frames, P))
            w = FeatureWindow(depth_threshold=4.0); arms["FeatureWindow"].append(run(w, frames, P)); w.close()
        dev = {}
        w = FeatureWindow(depth_threshold=4.0); run(w, frames, P, dev); w.close()        # a pass of its own: reading the events waits after every call
        out = {"features_per_frame": int(np.median([len(f) for f in frames])), "factors_per_window": arms["FeatureWindow"][0][2]}
        for arm, r in arms.items():
            fr, fl = [1e6 * x[0] for x in r], [1e6 * x[1] for x in r]
            out[arm] = {"stage_us": {"median": float(np.median(fr)), "min": min(fr), "max": max(fr)},
                        "factor_loop_us": {"median": float(np.median(fl)), "min": min(fl), "max": max(fl)}}
        out["FeatureWindow"]["device_us_per_operation"] = {k: {"median": 1e3 * float(np.median(v)), "max": 1e3 * float(np.max(v))} for k, v in dev.items()}
        out["c_abi"] = c_abi(frames, P, a.rounds)
        res[name] = out
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(json.dumps(res, indent=1) + "\n")


if __name__ == "__main__":
    main()
