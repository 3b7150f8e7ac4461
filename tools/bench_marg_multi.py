"""Batched marginalisations (gf_ba_marginalize_multi) against the two ways of serving K estimators without it, in one run.

Workloads (every window solved by the library first, as the reference marginalises at the optimum):
  c2_old            the C2 windows of bench.py, make_window(seed=100 + k), MARGIN_OLD: no prior, fast path
  wide_old          a chained window: solve -> MARGIN_OLD -> shift (frame 0 dropped, the prior attached) -> solve, with the speed
                    biases of frames 1..8 added to the prior (block-diagonal information 100).  The library's own chain keeps one
                    speed-bias block in the prior (n = 76 on these windows); the extra blocks make it wide enough for the literal
                    path: MARGIN_OLD keeps 133 columns (WIDE, Jacobi on the reduced system)
  wide_second_new   the same windows under MARGIN_SECOND_NEW (142 kept columns, WIDE)
For K in --ks:
  batched      one gf_ba_marginalize_multi call per round, K handles, one host thread
  sequential   K single calls per round on one handle
  threads      K handles, one host thread each making single calls (K <= 8)
Also: device ms per batch (CUDA events), a whole optimizationMulti round on c2 (solve_multi + marginalize_multi against
solve_multi + K single marginalisations; the blocks are restored before every round) and the largest scaled difference between
the batched and the single result of each window.  The card's name, power limit and max SM clock are read with nvidia-smi
(query only).  Prints one JSON line; --out also writes it.
  --profile DIR   instead: the kernel-by-kernel device time of one batch at K = 1 and K = 8 (torch.profiler, CUDA activities)
  --ab LIB        instead: the single call's device time on a c2 window and a wide_old window, alternating runs of this
                  library and of LIB (e.g. a build of the parent commit) in subprocesses; medians and spread"""
import argparse
import ctypes
import json
import os
import statistics
import subprocess
import sys
import threading
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from ground_fusion_b200._lib import MARGIN_OLD, MARGIN_SECOND_NEW, BaProblem  # noqa: E402
from ground_fusion_b200.ba_problem import Prior  # noqa: E402
from ground_fusion_b200.estimator import BundleAdjuster, solve_multi_structs  # noqa: E402
from ground_fusion_b200.synth_ba import make_window  # noqa: E402

BLOCKS = ("para_pose", "para_speed_bias", "para_feature", "para_ex_pose", "para_td")
WORKLOADS = ("c2_old", "wide_old", "wide_second_new")


def gpu_info():
    try:
        out = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], text=True)
        name, power, clock = [x.strip() for x in out.strip().splitlines()[0].split(",")]
        return {"name": name, "power_limit": power, "max_sm_clock": clock}
    except (OSError, subprocess.CalledProcessError, ValueError) as e:
        return {"error": str(e)}


def shifted(q, prior):
    """The window after MARGIN_OLD of q: frame 0 dropped, the rest kept, `prior` (already shifted by the library) attached."""
    nxt = q.clone(); nxt.n_frames = q.n_frames - 1
    nxt.para_pose = q.para_pose[1:].copy(); nxt.para_speed_bias = q.para_speed_bias[1:].copy()
    nxt.set_visual([(f.imu_i - 1, f.imu_j - 1, f.feature, list(f.pts_i), list(f.pts_j), list(f.vel_i), list(f.vel_j), f.td_i, f.td_j)
                    for f in list(q.visual)[:q.n_visual] if f.imu_i >= 1])
    nxt.set_imu([dict(i=f.i - 1, j=f.j - 1, sum_dt=f.sum_dt, delta_p=list(f.delta_p), delta_q=list(f.delta_q), delta_v=list(f.delta_v),
                      linearized_ba=list(f.linearized_ba), linearized_bg=list(f.linearized_bg),
                      jacobian=np.array(f.jacobian).reshape(15, 15), covariance=np.array(f.covariance).reshape(15, 15))
                 for f in list(q.imu)[1:q.n_imu]])
    nxt.prior = prior
    return nxt


def wide_window(ba, seed, sb_frames=range(1, 9), weight=100.0):
    q, _ = make_window(seed=seed)
    ba.optimization(q)
    pr = ba.marginalize_old(q)
    nxt = shifted(q, pr)
    extra = list(sb_frames)
    n0 = pr.n
    J = np.zeros((n0 + 9 * len(extra),) * 2)
    J[:n0, :n0] = pr.J
    J[n0:, n0:] = weight * np.eye(9 * len(extra))
    x0_len = sum({0: 7, 1: 9, 2: 7, 3: 1}[k] for k in pr.kinds)
    nxt.prior = Prior(pr.kinds + [1] * len(extra), pr.indices + extra, pr.idx + [n0 + 9 * j for j in range(len(extra))],
                      np.concatenate([pr.x0[:x0_len]] + [nxt.para_speed_bias[f] for f in extra]), J,
                      np.concatenate([pr.r, np.zeros(9 * len(extra))]))
    ba.optimization(nxt)
    return nxt


def build_windows(ba, workload, K):
    if workload == "c2_old":
        out = []
        for k in range(K):
            w = make_window(seed=100 + k)[0]
            ba.optimization(w)
            out.append(w)
        return out
    out, seed = [], 100
    while len(out) < K:      # MARGIN_SECOND_NEW needs para_Pose[WINDOW_SIZE - 1] in the prior: seeds whose chain lacks it are skipped
        w = wide_window(ba, seed)
        seed += 1
        if (0, w.n_frames - 2) in set(zip(w.prior.kinds, w.prior.indices)):
            out.append(w)
    return out


def mode_of(workload):
    return MARGIN_SECOND_NEW if workload.endswith("second_new") else MARGIN_OLD


class Calls:
    """ctypes arrays of one batch: the problems, modes, output buffers and result slots, built once for timing loops."""

    def __init__(self, wins, mode):
        from ground_fusion_b200._lib import BaPrior, lib
        self.L = lib()
        dp = ctypes.POINTER(ctypes.c_double)
        i32p = ctypes.POINTER(ctypes.c_int32)
        self.L.gf_ba_marginalize_multi.argtypes = [ctypes.POINTER(ctypes.c_void_p), ctypes.c_int, ctypes.POINTER(BaProblem), i32p,
                                                   ctypes.POINTER(BaPrior), ctypes.POINTER(dp), ctypes.POINTER(dp), ctypes.POINTER(dp),
                                                   i32p, ctypes.POINTER(ctypes.c_float)]
        fn = "gf_ba_marginalize_old" if mode == MARGIN_OLD else "gf_ba_marginalize_second_new"
        self.single_fn = getattr(self.L, fn)
        self.single_fn.argtypes = [ctypes.c_void_p, ctypes.POINTER(BaProblem), ctypes.POINTER(BaPrior), dp, dp, dp, ctypes.POINTER(ctypes.c_float)]
        K = len(wins)
        self.K = K
        self.structs = [w.struct() for w in wins]
        self.array = (BaProblem * K)(*self.structs)
        cap = 16 * 11 + 24
        self.bufs = [(np.zeros(cap), np.zeros(cap * cap), np.zeros(cap)) for _ in range(K)]
        self.ptrs = [(dp * K)(*[b[j].ctypes.data_as(dp) for b in self.bufs]) for j in range(3)]
        self.modes = np.full(K, mode, np.int32)
        self.outs = (BaPrior * K)()
        self.kept = np.zeros(K, np.int32)
        self.ms = ctypes.c_float(0)
        self.sbufs = [(np.zeros(cap), np.zeros(cap * cap), np.zeros(cap)) for _ in range(K)]
        self.souts = [BaPrior() for _ in range(K)]

    def batch(self, hs):
        harr = (ctypes.c_void_p * self.K)(*[h._h.value for h in hs])
        i32p = ctypes.POINTER(ctypes.c_int32)
        rc = self.L.gf_ba_marginalize_multi(harr, self.K, self.array, self.modes.ctypes.data_as(i32p), self.outs, self.ptrs[0], self.ptrs[1],
                                            self.ptrs[2], self.kept.ctypes.data_as(i32p), ctypes.byref(self.ms))
        assert rc == 0 and (self.kept > 0).all(), (rc, self.kept)
        return self.ms.value

    def single(self, h, k):
        dp = ctypes.POINTER(ctypes.c_double)
        b = self.sbufs[k]
        ms = ctypes.c_float(0)
        n = self.single_fn(h._h, ctypes.byref(self.structs[k]), ctypes.byref(self.souts[k]), b[0].ctypes.data_as(dp), b[1].ctypes.data_as(dp),
                           b[2].ctypes.data_as(dp), ctypes.byref(ms))
        assert n > 0, n
        return ms.value

    def max_scaled_diff(self):
        """Largest |H_batch - H_single| / sqrt(H_ii H_jj) and |b_batch - b_single| / max|b_single| over the windows (H = J0^T J0,
        b = J0^T r0: J0 is defined up to an orthogonal transform)."""
        worst = 0.0
        for k in range(self.K):
            n = int(self.kept[k])
            Jg, rg = self.bufs[k][1][:n * n].reshape(n, n), self.bufs[k][2][:n]
            Jw, rw = self.sbufs[k][1][:n * n].reshape(n, n), self.sbufs[k][2][:n]
            H, Hw = Jg.T @ Jg, Jw.T @ Jw
            worst = max(worst, float(np.abs((H - Hw) / (np.sqrt(np.outer(np.diag(Hw), np.diag(Hw))) + 1e-300)).max()))
            bw = Jw.T @ rw
            worst = max(worst, float(np.abs(Jg.T @ rg - bw).max() / np.abs(bw).max()))
        return worst


def run_k(workload, pool, K, rounds):
    c = Calls(pool[:K], mode_of(workload))
    hs = [BundleAdjuster(0) for _ in range(K)]
    single = BundleAdjuster(0)
    out = {"workload": workload, "K": K}
    try:
        for k in range(K):
            c.single(single, k)
        c.batch(hs)
        out["max_scaled_diff_vs_single"] = c.max_scaled_diff()
        dev = []
        t0 = time.perf_counter()
        for _ in range(rounds):
            dev.append(c.batch(hs))
        out["batched_margs_per_s"] = K * rounds / (time.perf_counter() - t0)
        out["device_ms_per_batch"] = statistics.median(dev)
        sdev = []
        t0 = time.perf_counter()
        for _ in range(rounds):
            sdev.append(sum(c.single(single, k) for k in range(K)))
        out["sequential_margs_per_s"] = K * rounds / (time.perf_counter() - t0)
        out["sequential_device_ms_sum"] = statistics.median(sdev)
        if K <= 8:
            def worker(k):
                for _ in range(rounds):
                    c.single(hs[k], k)
            th = [threading.Thread(target=worker, args=(k,)) for k in range(K)]
            t0 = time.perf_counter()
            for t in th:
                t.start()
            for t in th:
                t.join()
            out["threads_margs_per_s"] = K * rounds / (time.perf_counter() - t0)
    finally:
        for h in hs:
            h.close()
        single.close()
    return out


def run_round(pool, K, rounds):
    """A whole optimizationMulti round on c2: solve_multi, then the K marginalisations batched or one by one."""
    wins = [w.clone() for w in pool[:K]]
    saved = [[getattr(w, b).copy() for b in BLOCKS] for w in wins]
    c = Calls(wins, MARGIN_OLD)
    hs = [BundleAdjuster(0) for _ in range(K)]
    out = {"K": K}

    def restore():
        for w, s in zip(wins, saved):
            for b, v in zip(BLOCKS, s):
                getattr(w, b)[:] = v
    try:
        for label, marg in (("batched", lambda: c.batch(hs)), ("sequential", lambda: [c.single(hs[k], k) for k in range(K)])):
            restore(); solve_multi_structs(hs, c.array); marg()          # warm
            t0 = time.perf_counter()
            for _ in range(rounds):
                restore()
                sums, status = solve_multi_structs(hs, c.array)
                marg()
            out[label + "_rounds_per_s"] = rounds / (time.perf_counter() - t0)
    finally:
        for h in hs:
            h.close()
    return out


def profile(pools, out_dir):
    import torch
    from torch.profiler import ProfilerActivity
    torch.cuda.init()
    res = {}
    for workload in WORKLOADS:
        for K in (1, 8):
            c = Calls(pools[workload][:K], mode_of(workload))
            hs = [BundleAdjuster(0) for _ in range(K)]
            try:
                c.batch(hs); c.batch(hs)                                 # warm
                with torch.profiler.profile(activities=[ProfilerActivity.CUDA]) as prof:
                    c.batch(hs)
                    torch.cuda.synchronize()
            finally:
                for h in hs:
                    h.close()
            rows = []
            for e in prof.key_averages():
                us = getattr(e, "device_time_total", None)
                if us is None:
                    us = e.cuda_time_total
                if us > 0:
                    rows.append({"name": e.key, "calls": e.count, "device_us": round(us, 2)})
            rows.sort(key=lambda r: -r["device_us"])
            key = "%s_K%d" % (workload, K)
            res[key] = {"device_ms_event": c.ms.value, "kernels": rows}
            prof.export_chrome_trace(os.path.join(out_dir, key + ".pt.trace.json"))
    return res


def single_times(reps):
    """Median device ms of the single call on a c2 window and on a wide_old window (the library GF_B200_LIB selects)."""
    ba = BundleAdjuster(0)
    try:
        c2 = build_windows(ba, "c2_old", 1)[0]
        wide = build_windows(ba, "wide_old", 1)[0]
        out = {}
        for name, w in (("c2_old", c2), ("wide_old", wide)):
            for _ in range(3):
                ba.marginalize_old(w)
            t = []
            for _ in range(reps):
                ba.marginalize_old(w)
                t.append(ba.last_marg_ms)
            out[name] = statistics.median(t)
        return out
    finally:
        ba.close()


def ab(other_lib, runs, reps):
    here = os.path.abspath(__file__)
    libs = {"this": None, "other": os.path.abspath(other_lib)}
    res = {k: {"c2_old": [], "wide_old": []} for k in libs}
    for r in range(runs):
        for name in (("this", "other") if r % 2 == 0 else ("other", "this")):
            env = dict(os.environ)
            env.pop("GF_B200_LIB", None)
            if libs[name]:
                env["GF_B200_LIB"] = libs[name]
            line = subprocess.check_output([sys.executable, here, "--single-times", str(reps)], env=env, text=True).strip().splitlines()[-1]
            for k, v in json.loads(line).items():
                res[name][k].append(v)
    summary = {}
    for name, d in res.items():
        summary[name] = {k: {"median_ms": statistics.median(v), "min_ms": min(v), "max_ms": max(v), "runs": v} for k, v in d.items()}
    return summary


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ks", default="1,2,4,8,16,32,64")
    ap.add_argument("--margs", type=int, default=256, help="marginalisations per method and K (rounds = max(3, margs / K))")
    ap.add_argument("--out", default=None)
    ap.add_argument("--profile", default=None, metavar="DIR")
    ap.add_argument("--ab", default=None, metavar="LIB")
    ap.add_argument("--ab-runs", type=int, default=6)
    ap.add_argument("--single-times", type=int, default=0, help=argparse.SUPPRESS)
    a = ap.parse_args()
    if a.single_times:
        print(json.dumps(single_times(a.single_times)))
        return
    if a.ab:
        res = {"metric": "single_marginalisation_device_ms", "gpu": gpu_info(), "ab_runs": a.ab_runs, "reps_per_run": 50,
               "note": "median over 50 calls per run, runs alternate between the two libraries", "results": ab(a.ab, a.ab_runs, 50)}
        line = json.dumps(res)
        print(line)
        if a.out:
            with open(a.out, "w") as f:
                f.write(line + "\n")
        return
    ks = [int(x) for x in a.ks.split(",")]
    ba = BundleAdjuster(0)
    try:
        pools = {w: build_windows(ba, w if w != "wide_second_new" else "wide_old", max(ks) if not a.profile else 8) for w in WORKLOADS[:2]}
    finally:
        ba.close()
    pools["wide_second_new"] = pools["wide_old"]
    if a.profile:
        os.makedirs(a.profile, exist_ok=True)
        res = {"metric": "marginalisation_kernel_split", "gpu": gpu_info(), "profiles": profile(pools, a.profile)}
        line = json.dumps(res)
        print(line)
        with open(os.path.join(a.profile, "marg_multi_kernels.json"), "w") as f:
            f.write(line + "\n")
        return
    run_k("c2_old", pools["c2_old"], 2, 3)                        # warm-up: module load, buffer growth, first launches
    rows = []
    for workload in WORKLOADS:
        for K in ks:
            rows.append(run_k(workload, pools[workload], K, max(3, a.margs // K)))
    rounds = [run_round(pools["c2_old"], K, max(3, a.margs // K)) for K in ks]
    res = {"metric": "ba_multi_marginalisations_per_sec", "unit": "marginalisations/s", "gpu": gpu_info(),
           "workloads": {"c2_old": "make_window(seed=100+k) solved, MARGIN_OLD, no prior (fast path)",
                         "wide_old": "solve -> MARGIN_OLD -> shift -> solve of make_window(seed=100+k), prior widened by the speed biases "
                                     "of frames 1..8: 133 kept (literal path, WIDE)",
                         "wide_second_new": "the wide_old windows under MARGIN_SECOND_NEW: 142 kept (WIDE)"},
           "rows": rows, "optimization_multi_rounds": rounds}
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
