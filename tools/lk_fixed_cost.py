"""Splits k_track's per-feature time into a fixed part and a part per LK iteration.

Runs the C2 synthetic stream (640x480, 150 features) and reads, for every tracked feature of every frame, the clock64
cycles of its whole track_point (forward pass, reverse check, border tests) and its LK iteration count
(gf_tracker_debug_read, [64 + 8*i] and [64 + 8*i + 1]).  A least-squares fit cycles = a + b * iterations then gives a,
the fixed cost per feature (prologue and the setup of every pyramid level it does not hide), and b, the cost of one
iteration.  Also prints the slowest feature per frame, which sets k_track's time for one stream, and the mean clock64
phase counters of features 0..3 ([32 + 8*i + k], the LKP marks of fe_lk.cuh).

The counters are compiled in only with -DGF_PROFILE: run `make profile` first; the tool loads
ground_fusion_b200/libgf_b200_prof.so unless GF_B200_LIB names another library.

    python tools/lk_fixed_cost.py [--features 4000] [--out FILE]
"""
import argparse
import ctypes
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
os.environ.setdefault("GF_B200_LIB", os.path.join(ROOT, "ground_fusion_b200", "libgf_b200_prof.so"))
from ground_fusion_b200._lib import lib  # noqa: E402
from ground_fusion_b200.feature_tracker import FeatureTracker  # noqa: E402
from ground_fusion_b200.synth import SyntheticStream, idc_params8  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--features", type=int, default=4000, help="stop after this many tracked features")
    ap.add_argument("--warmup", type=int, default=3, help="frames run before counting")
    ap.add_argument("--out", default=None, help="also write the JSON result here")
    args = ap.parse_args()

    import torch
    dev = torch.cuda.get_device_name(0)
    st = SyntheticStream(seed=0)
    tr = FeatureTracker(640, 480, idc_params8(), 150, 30, 1, 1)
    N = 64 + 8 * 1024
    buf = (ctypes.c_longlong * N)()
    cyc, its, frame_max, phases = [], [], [], []
    k = 0
    while len(cyc) < args.features:
        t, g, d = st.frame(k)
        tr.trackImageRaw(t, g, d)
        n = int(tr.last_info["n_prev"])
        if k >= args.warmup and n > 0:
            assert lib().gf_tracker_debug_read(tr._h, buf, N) == 0
            dbg = np.array(buf[:], dtype=np.int64)
            lk = dbg[64:64 + 8 * n].reshape(n, 8)
            phases.append(dbg[32:32 + 8 * min(n, 4)].reshape(-1, 8).mean(0))
            cyc.extend(lk[:, 0].tolist())
            its.extend(lk[:, 1].tolist())
            frame_max.append(int(lk[:, 0].max()))
        k += 1
    tr.close()
    cyc = np.array(cyc, dtype=np.float64)
    if not cyc.any():
        sys.exit("all cycle counters are 0: %s was built without -DGF_PROFILE" % os.environ["GF_B200_LIB"])
    its = np.array(its, dtype=np.float64)
    b, a = np.polyfit(its, cyc, 1)
    resid = cyc - (a + b * its)
    res = {
        "device": dev,
        "frames": k - args.warmup,
        "features": int(cyc.size),
        "fit_a_cycles": round(float(a), 1),
        "fit_b_cycles_per_iteration": round(float(b), 1),
        "fit_rms_cycles": round(float(np.sqrt(np.mean(resid ** 2))), 1),
        "iterations_mean": round(float(its.mean()), 2),
        "cycles_mean": round(float(cyc.mean()), 1),
        "cycles_p50": float(np.median(cyc)),
        "slowest_feature_cycles_median_over_frames": float(np.median(frame_max)),
        "phase_cycles_features_0_3": [round(float(v), 1) for v in np.mean(phases, 0)],
    }
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
