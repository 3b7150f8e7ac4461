"""The FeatureManager stage of K estimators: gf_fm_window_group (one set of launches per call for all K) against K single
gf_fm_window handles called in sequence and K handles on K threads.

The stage is what one processImage does around the solve (as tools/bench_fm_window.py times it for one window): add_frame,
triangulate, fill_problem, set_depth, the consistency check and removal, predict_next, the slide's removal and
remove_failures.  Every member gets the C2 replay frames (150 features per frame).  Fields of the result:
  c_abi               host time per round (one frame of every member) from C++ alone (adaptor/harness fm-group-bench), the three
                      arms alternating in one process over --rounds passes: median, min, max, for K in --ks
  python              the same from Python (FeatureWindowGroup against K FeatureWindows in sequence), for reference
  device_ms_per_call  CUDA-event time of each group call at K = 8 (gf_fm_window_group_last_device_ms)
  launches_per_round  CUDA kernels per steady-state round at K = 1 and K = 8, from torch.profiler in a pass of its own
  replay_group        seconds per frame of one replay_group run at K = 8 against K independent replay() loops
  single_window       the one-window stage (harness fm-bench, gf_fm_window arm) of this tree and of --parent (a directory with the
                      parent commit's adaptor/_build/harness and ground_fusion_b200/libgf_b200.so), alternating, with the spread
  card                name and power limit of the GPU, read in the same run
Needs a GPU: there is no CPU fallback.

    python tools/bench_fm_group.py --out profiles/h100_fm_group_c2.json [--parent DIR]
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

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_fm_window import c2_frames, poses                          # noqa: E402
from ground_fusion_b200.ba_problem import Problem                     # noqa: E402
from ground_fusion_b200.feature_window import FeatureWindow, FeatureWindowGroup   # noqa: E402
from ground_fusion_b200 import _lib                                   # noqa: E402


def write_input(path, frames, P, rounds, ks=None):
    Ps, Rs, tic, ric = P
    with open(path, "wb") as f:
        f.write(struct.pack("<2i2d33d99d3d9d", rounds, len(frames), 10.0 / 600.0, 4.0, *Ps.ravel(), *Rs.ravel(), *tic, *ric.ravel()))
        for fr in frames:
            f.write(struct.pack("<i", len(fr)) + b"".join(struct.pack("<i8d", k, *fr[k][:8]) for k in sorted(fr)))
        if ks is not None:
            f.write(struct.pack("<i%di" % len(ks), len(ks), *ks))


def harness(root, mode, inp, tmp, tag):
    out = os.path.join(tmp, tag + ".json")
    subprocess.check_call([os.path.join(root, "adaptor", "_build", "harness"), mode, inp, out])
    return json.load(open(out))


def c_abi(frames, P, rounds, ks, tmp):
    subprocess.check_call(["make", "-s", "-C", os.path.join(ROOT, "adaptor")])
    inp = os.path.join(tmp, "group.bin")
    write_input(inp, frames, P, rounds, ks)
    return harness(ROOT, "fm-group-bench", inp, tmp, "group")


def single_window(frames, P, rounds, parent, tmp):
    """harness fm-bench of this tree and of the parent, alternating; the gf_fm_window arm's stage time per pass."""
    inp = os.path.join(tmp, "single.bin")
    write_input(inp, frames, P, 1)
    arms = {"this_tree": ROOT, "parent": parent}
    out = {k: [] for k in arms}
    for _ in range(rounds):
        for k, root in arms.items():
            out[k].append(harness(root, "fm-bench", inp, tmp, k)["gf_fm_window"]["stage_us"]["median"])
    return {k: {"median": float(np.median(v)), "min": min(v), "max": max(v), "passes": v} for k, v in out.items()}


def py_stage(members, grp, frames, P, device_ms=None):
    """One pass of the stage from Python, the group (grp) or the members in sequence (grp None); seconds per round."""
    Ps, Rs, tic, ric = P
    K = len(members)
    obs = []
    for image in frames:
        o = np.zeros(len(image), _lib.OBS_DTYPE)
        ids = sorted(image)
        o["id"] = ids; o["v"] = np.asarray([image[i][:8] for i in ids])
        obs.append(o)
    for w in members:
        w.clearState()

    def dev(name):
        if device_ms is not None:
            device_ms.setdefault(name, []).append(grp.last_device_ms())

    t0 = time.perf_counter()
    for k, o in enumerate(obs):
        fc = min(k, 10)
        if grp is None:
            for w in members:
                margin = w.addFrame(fc, o, None, 0.0)
                if fc < 10:
                    continue
                w.triangulateAll(fc, Ps, Rs, tic, ric)
                pb = Problem(11, 0); n = w.fillProblem(pb)
                w.setDepth(pb.para_feature[:n])
                w.removeOutlier(set(sorted(w.movingConsistencyCheckW(Ps, Rs, tic, ric))[:3]))
                w.predictPtsInNextFrame(fc, Ps, Rs, tic, ric)
                if margin or k % 3 == 0:
                    w.removeBackShiftDepth(Rs[0], Ps[0], Rs[1], Ps[1])
                else:
                    w.removeFront(fc)
                w.removeFailures()
                w.size()
            continue
        margins = grp.addFrames([fc] * K, [o] * K, None, [0.0] * K); dev("add_frame")
        if fc < 10:
            continue
        ps = [(Ps, Rs, tic, ric)] * K
        grp.triangulateAll([fc] * K, ps); dev("triangulate")
        pbs = [Problem(11, 0) for _ in range(K)]
        nf = grp.fillProblems(pbs); dev("fill_problem")
        grp.setDepths([pb.para_feature[:n] for pb, n in zip(pbs, nf)]); dev("set_depth")
        bad = grp.movingConsistencyCheckW(ps); dev("outliers")
        grp.removeOutliers([set(sorted(b)[:3]) for b in bad]); dev("remove_ids")
        grp.predictPtsInNextFrame([fc] * K, ps); dev("predict_next")
        ops = [_lib.FM_REMOVE_BACK_SHIFT_DEPTH if (m or k % 3 == 0) else _lib.FM_REMOVE_FRONT for m in margins]
        grp.remove(ops, [fc] * K, [(Rs[0], Ps[0], Rs[1], Ps[1])] * K); dev("remove")
        grp.removeFailures(); dev("remove_failures")
        grp.last_device_ms()
    return (time.perf_counter() - t0) / len(frames)


def python_arms(frames, P, rounds, ks):
    out = {}
    for K in ks:
        ws = [FeatureWindow(depth_threshold=4.0) for _ in range(K)]
        grp = FeatureWindowGroup(ws)
        py_stage(ws, grp, frames, P); py_stage(ws, None, frames, P)          # warm-up
        g, s = [], []
        for _ in range(rounds):
            g.append(1e6 * py_stage(ws, grp, frames, P)); s.append(1e6 * py_stage(ws, None, frames, P))
        out[str(K)] = {"group": {"median": float(np.median(g)), "min": min(g), "max": max(g)},
                       "sequential": {"median": float(np.median(s)), "min": min(s), "max": max(s)}}
        grp.close()
        for w in ws:
            w.close()
    return out


def device_ms(frames, P, K=8):
    ws = [FeatureWindow(depth_threshold=4.0) for _ in range(K)]
    grp = FeatureWindowGroup(ws)
    d = {}
    py_stage(ws, grp, frames, P, d)
    grp.close()
    for w in ws:
        w.close()
    return {k: {"median": float(np.median(v)), "max": float(np.max(v))} for k, v in d.items()}


def launches(frames, P, ks=(1, 8)):
    """CUDA kernels per steady-state round of the group stage, counted by torch.profiler over one pass."""
    from torch.profiler import ProfilerActivity, profile
    out = {}
    rounds = sum(1 for k in range(len(frames)) if k >= 10)
    for K in ks:
        ws = [FeatureWindow(depth_threshold=4.0) for _ in range(K)]
        grp = FeatureWindowGroup(ws)
        py_stage(ws, grp, frames, P)
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            py_stage(ws, grp, frames, P)
        names = [e.name for e in prof.events() if e.device_type.name == "CUDA" and "k_fmw" in e.name]
        fill = sum(1 for k in range(len(frames)) if k < 10)
        out[str(K)] = {"kernels_in_pass": len(names), "fill_frames": fill, "steady_rounds": rounds,
                       "kernels_per_steady_round": (len(names) - fill) / rounds}
        grp.close()
        for w in ws:
            w.close()
    return out


def replay_round(n, K=8):
    from ground_fusion_b200.estimator import BundleAdjuster
    from ground_fusion_b200.feature_tracker import FeatureTracker
    from ground_fusion_b200.replay import replay, replay_group
    from ground_fusion_b200.synth import IDC_CAM, SyntheticStream
    cam = dict(IDC_CAM, k1=0.0, k2=0.0, p1=0.0, p2=0.0)
    p8 = [cam[k] for k in ("fx", "fy", "cx", "cy", "k1", "k2", "p1", "p2")]

    def parts():
        return ([FeatureTracker(640, 480, p8, 150, 30, 1, 1) for _ in range(K)], [FeatureWindow(depth_threshold=4.0) for _ in range(K)],
                [BundleAdjuster(0) for _ in range(K)])
    trs, ws, bas = parts()
    t0 = time.perf_counter()
    replay_group([SyntheticStream(seed=s) for s in range(K)], trs, ws, bas, n)
    tg = (time.perf_counter() - t0) / n
    for x in trs + ws + bas:
        x.close()
    trs, ws, bas = parts()
    t0 = time.perf_counter()
    for s in range(K):
        replay(SyntheticStream(seed=s), trs[s], ws[s], bas[s], n)
    ti = (time.perf_counter() - t0) / n
    for x in trs + ws + bas:
        x.close()
    return {"K": K, "frames": n, "replay_group_s_per_frame": tg, "independent_replays_s_per_frame": ti,
            "note": "wall time per frame of all K streams, initialisation frames included; one run each"}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=64)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--ks", default="1,2,4,8,16,32,64")
    ap.add_argument("--py-ks", default="1,2,4,8")
    ap.add_argument("--replay-frames", type=int, default=32)
    ap.add_argument("--parent", default=None, help="directory with the parent commit's adaptor/_build/harness and ground_fusion_b200/libgf_b200.so")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_fm_group needs a GPU")
    card = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"]).decode().strip()
    P = poses()
    frames = c2_frames(a.frames)
    ks = [int(x) for x in a.ks.split(",")]
    res = {"card": card, "stream": "c2 replay frames, %d per member" % int(np.median([len(f) for f in frames])), "frames": a.frames,
           "rounds": a.rounds}
    with tempfile.TemporaryDirectory() as tmp:
        res["c_abi"] = c_abi(frames, P, a.rounds, ks, tmp)
        res["single_window"] = single_window(frames, P, a.rounds, a.parent, tmp) if a.parent else "not measured (no --parent)"
    res["python"] = python_arms(frames, P, a.rounds, [int(x) for x in a.py_ks.split(",")])
    res["python"]["unit"] = "microseconds of host time per round, mean over a pass"
    res["device_ms_per_call"] = device_ms(frames, P)
    res["launches_per_round"] = launches(frames, P)
    res["replay_group"] = replay_round(a.replay_frames)
    res["card_after"] = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"]).decode().strip()
    print(json.dumps(res))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(json.dumps(res, indent=1) + "\n")


if __name__ == "__main__":
    main()
