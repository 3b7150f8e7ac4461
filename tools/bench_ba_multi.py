"""Batched sliding-window solves (gf_ba_solve_multi) against the two ways of serving K estimators without it, in one run.

For K in --ks, on the C2 windows of bench.py (make_window(seed=100 + k)):
  batched      one gf_ba_solve_multi call per round, K handles, one host thread
  sequential   K gf_ba_solve calls per round on one handle
  threads      K handles, one host thread each calling gf_ba_solve (K <= 8)
Every round restores the windows' blocks first (as bench.py does), so all three include the same host work.  Also reported:
device ms per batch (CUDA events), a whole-program FP64 rate -- algorithmic FLOPs over the batch's device time, against the
DMMA peak gf_probe_fp64 measures in the same run -- and the largest difference between the batched and the single solve of each
window.  The card's name and power limit are read with nvidia-smi (query only).  Prints one JSON line; --out also writes it."""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import threading
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from ground_fusion_b200 import _lib  # noqa: E402
from ground_fusion_b200._lib import BaProblem  # noqa: E402
from ground_fusion_b200.estimator import BundleAdjuster, solve_multi_structs  # noqa: E402
from ground_fusion_b200.synth_ba import make_window  # noqa: E402

BLOCKS = ("para_pose", "para_speed_bias", "para_feature", "para_ex_pose", "para_td")


def gpu_info():
    try:
        out = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], text=True)
        name, power, clock = [x.strip() for x in out.strip().splitlines()[0].split(",")]
        return {"name": name, "power_limit": power, "max_sm_clock": clock}
    except (OSError, subprocess.CalledProcessError, ValueError) as e:
        return {"error": str(e)}


class Windows:
    def __init__(self, K):
        self.w = [make_window(seed=100 + k)[0] for k in range(K)]
        self.saved = [[getattr(w, b).copy() for b in BLOCKS] for w in self.w]
        self.structs = [w.struct() for w in self.w]
        self.array = (BaProblem * K)(*self.structs)       # copies of the structs: same pointers into the windows' arrays

    def restore(self, k):
        for b, v in zip(BLOCKS, self.saved[k]):
            getattr(self.w[k], b)[:] = v


def step_flops(nc, n_lm):
    """Algorithmic FP64 FLOPs of one k_ba_step launch that takes a step (bench.py's formula: factorisation, two triangular
    solves, landmark back substitution and dogleg terms) plus the rank-L update of the reduced system in k_ba_schur."""
    fma = (nc + 1) ** 3 / 3.0 + nc * nc + 3.0 * n_lm * nc + n_lm * (nc + 1) * (nc + 2) / 2.0
    return 2.0 * fma


def run_k(K, rounds, L):
    ws = Windows(K)
    hs = [BundleAdjuster(0) for _ in range(K)]
    prof = (ctypes.c_longlong * 32)()
    out = {"K": K}
    try:
        # correctness at this size: batched against single solves of the same windows
        single = BundleAdjuster(0)
        want = []
        for k in range(K):
            ws.restore(k); single.solve_struct(ws.structs[k])
            want.append([getattr(ws.w[k], b).copy() for b in BLOCKS])
        for k in range(K):
            ws.restore(k)
        sums, status = solve_multi_structs(hs, ws.array)
        assert (status == 0).all()
        out["max_abs_diff_vs_single"] = max(float(np.abs(getattr(ws.w[k], b) - v).max()) for k in range(K) for b, v in zip(BLOCKS, want[k]))
        # batched
        dev_ms, flops = 0.0, 0.0
        t0 = time.perf_counter()
        for _ in range(rounds):
            for k in range(K):
                ws.restore(k)
            sums, status = solve_multi_structs(hs, ws.array)
            dev_ms += sums[0].device_ms
        el = time.perf_counter() - t0
        for k in range(K):             # step launches of the last round, per window
            L.gf_ba_debug_profile(hs[k]._h, prof)
            flops += step_flops(int(sums[k].reduced_dim), int(sums[k].n_free_landmarks)) * prof[31]
        out["batched_solves_per_s"] = K * rounds / el
        out["device_ms_per_batch"] = dev_ms / rounds
        out["fp64_gflops_whole_solve"] = flops / (sums[0].device_ms * 1e-3) / 1e9
        # K sequential gf_ba_solve on one handle
        t0 = time.perf_counter()
        for _ in range(rounds):
            for k in range(K):
                ws.restore(k); single.solve_struct(ws.structs[k])
        out["sequential_solves_per_s"] = K * rounds / (time.perf_counter() - t0)
        single.close()
        # K handles, K threads
        if K <= 8:
            def worker(k):
                for _ in range(rounds):
                    ws.restore(k); hs[k].solve_struct(ws.structs[k])
            th = [threading.Thread(target=worker, args=(k,)) for k in range(K)]
            t0 = time.perf_counter()
            for t in th:
                t.start()
            for t in th:
                t.join()
            out["threads_solves_per_s"] = K * rounds / (time.perf_counter() - t0)
    finally:
        for h in hs:
            h.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ks", default="1,2,4,8,16,32,64,128")
    ap.add_argument("--solves", type=int, default=400, help="solves per method and K (rounds = max(3, solves / K))")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    L = _lib.lib()
    L.gf_ba_debug_profile.argtypes = [ctypes.c_void_p, ctypes.POINTER(ctypes.c_longlong)]
    L.gf_probe_fp64.argtypes = [ctypes.c_int, ctypes.POINTER(ctypes.c_double), ctypes.POINTER(ctypes.c_double)]
    dfma, dmma = ctypes.c_double(0), ctypes.c_double(0)
    _lib.check(L.gf_probe_fp64(0, ctypes.byref(dfma), ctypes.byref(dmma)))
    ks = [int(x) for x in a.ks.split(",")]
    run_k(2, 3, L)                                     # warm-up: module load, buffer growth, first launches
    rows = []
    for K in ks:
        r = run_k(K, max(3, a.solves // K), L)
        r["fp64_frac_of_dmma_peak"] = r["fp64_gflops_whole_solve"] / dmma.value
        rows.append(r)
    res = {"metric": "ba_multi_solves_per_sec", "unit": "solves/s", "workload": "C2 windows make_window(seed=100+k), max 8 iterations",
           "gpu": gpu_info(), "dmma_peak_gflops": dmma.value, "dfma_peak_gflops": dfma.value,
           "fp64_note": "whole-program figure: algorithmic FLOPs of every step-taking k_ba_step launch (factorisation, solves, "
                        "landmark terms) and the Schur rank-L update, over the batch's device time; peak = gf_probe_fp64 DMMA, this run",
           "rows": rows}
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
