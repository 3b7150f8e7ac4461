"""Compares two `bench.py --dump-outputs` directories byte for byte.

    python tools/compare_dumps.py DIR_A DIR_B [--ignore-info FIELD ...]

Every .npy array must be identical in dtype, shape and bytes (NaN padding included).  --ignore-info drops the named
gf_track_info columns of fe_info first (e.g. nms_rounds, which counts the rounds of the min-distance pass, not its result).
Exit status 0 when everything matches.
"""
import argparse
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

INFO_FIELDS = ("n_prev", "n_tracked", "n_kept", "n_new", "n_candidates", "nms_rounds", "eig_fixups", "lk_iterations")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("a")
    ap.add_argument("b")
    ap.add_argument("--ignore-info", nargs="*", default=[], choices=INFO_FIELDS)
    args = ap.parse_args()
    names = sorted(f for f in os.listdir(args.a) if f.endswith(".npy"))
    if names != sorted(f for f in os.listdir(args.b) if f.endswith(".npy")):
        print("different file sets"); return 1
    bad = 0
    for f in names:
        x, y = np.load(os.path.join(args.a, f)), np.load(os.path.join(args.b, f))
        if f == "fe_info.npy" and args.ignore_info:
            keep = [i for i, n in enumerate(INFO_FIELDS) if n not in args.ignore_info]
            x, y = x[:, keep], y[:, keep]
        same = x.dtype == y.dtype and x.shape == y.shape and x.tobytes() == y.tobytes()
        print("%-24s %s %s" % (f, x.shape, "identical" if same else "DIFFERENT"))
        bad += not same
    return 1 if bad else 0


if __name__ == "__main__":
    sys.exit(main())
