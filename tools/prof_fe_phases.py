"""Prints the clock64 phase counters of the FE kernels (gf_tracker_debug_read) over a few C2 frames."""
import sys, os, ctypes
import numpy as np
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from ground_fusion_b200.feature_tracker import FeatureTracker
from ground_fusion_b200._lib import lib
from ground_fusion_b200.synth import SyntheticStream
from ground_fusion_b200.synth import idc_params8
st = SyntheticStream(seed=0)
tr = FeatureTracker(640, 480, idc_params8(), 150, 30, 1, 1)
n = int(sys.argv[1]) if len(sys.argv) > 1 else 12
N = 64 + 8 * 150
buf = (ctypes.c_longlong * N)()
for k in range(n):
    t, g, d = st.frame(k)
    tr.trackImageRaw(t, g, d)
    lib().gf_tracker_debug_read(tr._h, buf, N)
    a = np.array(buf[:], dtype=np.int64)
    lk = a[64:].reshape(-1, 8)
    cyc, it = lk[:, 0], lk[:, 1]
    fast, slow = lk[:tr.last_info["n_prev"], 2:4].sum(0)      # rows past n_prev are stale
    print(f"frame {k}: dev {tr.last_device_ms():.3f} ms info {tr.last_info}")
    print(f"   lk b sums: {fast} iterations from the integer partials, {slow} from the sequential chains"
          f" ({100.0 * fast / max(fast + slow, 1):.1f} % fast)")
    print(f"   setmask cyc: compact {a[0]} sort {a[1]} greedy {a[2]} emit {a[3]}")
    print(f"   finalize cyc: nms {a[8]} topk {a[9]} emit {a[10]}  nacc {a[11]} ncand {a[12]}")
    print(f"   nms detail: setup {a[16]} A {a[13]} B {a[14]} C {a[15]} total {a[17]}")
    print(f"   lk: cyc max {cyc.max()} mean {cyc.mean():.0f} p50 {np.median(cyc):.0f}  iters max {it.max()} mean {it.mean():.1f};"
          f" cyc/iter (top5 by cyc) {[ (int(c), int(i)) for c, i in sorted(zip(cyc, it), reverse=True)[:5]]}")
    for f in range(2):
        pc = a[32 + 8 * f: 40 + 8 * f]
        print(f"   lk feature {f}: total {lk[f,0]} iters {lk[f,1]} | stageI {pc[0]} scharr {pc[1]} bilin {pc[2]} chainA+stageJ {pc[3]} postA {pc[4]} | iter: terms {pc[5]} chain {pc[6]} rest {pc[7]}")
