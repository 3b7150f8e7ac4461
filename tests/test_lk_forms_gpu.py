"""GPU tests of what the choice between the two LK forms adds (run with -m gpu on an H100).

A tracker runs k_track / k_lk_pred in the two-role form (fe_lk.cuh) while it is the only live tracker on its device and in
the single-role form (fe_lk_single.cuh) while others are live; tracker groups always take the single-role form
(DESIGN.md §1.3).  The form is chosen when a frame is enqueued, and each (frame % 6, prediction, form) has its own
captured graph.  These tests check that both forms agree in everything the tracker reports, that a tracker switching
form mid-stream (a companion tracker created or closed, also with frames in flight) stays bit-exact with
oracle/fe_oracle.py, and both forms on the largest b-term partials an 8-bit image allows.
"""
import gc

import numpy as np
import pytest

from test_fe_edges_gpu import check_lk
from test_fe_gpu import check_form, check_oracle, lk_debug, lk_form  # noqa: F401 (fixture)
from test_lk_overlap_gpu import min_eig, window_terms

pytestmark = pytest.mark.gpu
cv2 = pytest.importorskip("cv2")


def _cam():
    from oracle.fe_oracle import IDC_CAM, PinholeCamera
    return PinholeCamera(**IDC_CAM)


def _tracker(gf):
    return gf.FeatureTracker(640, 480, _cam().params8(), 150, 30, 1, 1)


def _frames(seed, n, stretch=()):
    """n frames of SyntheticStream(seed); the gray frames with index in `stretch` are stretched 5x about 128 and clipped,
    so that many b chains leave the integer path's bound."""
    from ground_fusion_b200.synth import SyntheticStream
    st = SyntheticStream(seed=seed)
    out = []
    for k in range(n):
        t, g, d = st.frame(k)
        if k in stretch:
            g = np.clip((g.astype(np.int32) - 128) * 5 + 128, 0, 255).astype(np.uint8)
        out.append((t, np.ascontiguousarray(g), np.ascontiguousarray(d)))
    return out


def _prediction(obs, rng, every=1):
    """setPrediction input from a frame's observations: the ray times its depth, slightly perturbed."""
    pred = {}
    for o in obs[::every]:
        d = max(o["v"][7], 0.5)
        pred[int(o["id"])] = (o["v"][0] * d + rng.normal(0, 0.002), o["v"][1] * d + rng.normal(0, 0.002), d)
    return pred


def test_forms_agree_in_iterations_and_paths(gf):
    """The same stream through a lone tracker and through one with a companion: per frame the observations, ids, status and
    last_info (the LK iteration total included) are equal, and per feature so are the iteration count and its split between
    the integer path and the chain path, which the oracle cannot see when the final point is the same.  The stream has a
    clipped high-contrast stretch, a setPrediction frame (k_lk_pred) and a removeOutliers frame."""
    frames = _frames(13, 20, stretch=range(7, 13))
    runs = {}
    for form in ("two-role", "single-role"):
        gc.collect()
        companion = _tracker(gf) if form == "single-role" else None
        tr = _tracker(gf)
        rng = np.random.default_rng(3)
        rows = []
        for k, (t, g, d) in enumerate(frames):
            obs = tr.trackImageRaw(t, g, d).copy()
            check_form(k, tr, form)
            rows.append((obs.tobytes(), tr.last_status.copy(), dict(tr.last_info), lk_debug(tr)[:, 1:4]))
            if k in (4, 10):
                tr.setPrediction(_prediction(obs, rng))
            if k in (5, 14):
                tr.removeOutliers(set(int(i) for i in obs["id"][::6]))
        tr.close()
        if companion is not None:
            companion.close()
        runs[form] = rows
    paths = np.zeros(2, np.int64)
    for k, (a, b) in enumerate(zip(runs["two-role"], runs["single-role"])):
        assert a[2] == b[2], "frame %d: %s vs %s" % (k, a[2], b[2])
        assert np.array_equal(a[1], b[1]), "frame %d: status" % k
        assert a[0] == b[0], "frame %d: observations" % k
        bad = np.flatnonzero(np.any(a[3] != b[3], 1))
        assert not len(bad), "frame %d feature %d: iterations / integer / chain %s vs %s" % (k, bad[0], a[3][bad[0]], b[3][bad[0]])
        paths += a[3][:, 1:3].sum(0)
    assert paths[0] > 0 and paths[1] > 0, paths


@pytest.mark.parametrize("mode", ["graph", "direct"])
def test_form_switches_during_a_stream(gf, monkeypatch, mode):
    """One tracker against the oracle, bit for bit, while a companion tracker is created (frames 6..11 and 18..23 run the
    single-role form) and closed (frames 12..17 two-role again).  A setPrediction before frames 3, 9, 15 and 21, which
    share the graph key frame % 6 = 3: each (prediction, form) graph is captured in the first two blocks of six frames
    and replayed after a switch in the last two.  Direct mode (GF_NO_GRAPH, read when the tracker is created) launches
    the same kernels without graphs."""
    from oracle.fe_oracle import FeatureTrackerOracle
    if mode == "direct":
        monkeypatch.setenv("GF_NO_GRAPH", "1")
    else:
        monkeypatch.delenv("GF_NO_GRAPH", raising=False)
    gc.collect()
    gpu = _tracker(gf)
    ref = FeatureTrackerOracle(_cam(), 150, 30, 1, 1)
    rng = np.random.default_rng(5)
    companion = None
    for k, (t, g, d) in enumerate(_frames(14, 24)):
        if k % 6 == 0 and (k // 6) % 2 == 1:
            companion = _tracker(gf)
        elif k % 6 == 0 and companion is not None:
            companion.close()
            companion = None
        got = gpu.trackImageRaw(t, g, d)
        want = ref.trackImage(t, g, d)
        check_oracle(k, gpu, got, ref, want)
        check_form(k, gpu, "single-role" if companion is not None else "two-role")
        if k % 6 == 2:
            pred = _prediction(got, rng, every=2)
            gpu.setPrediction(pred)
            ref.setPrediction(pred)
    assert companion is not None
    companion.close()
    gpu.close()


def test_form_switch_with_frames_in_flight(gf):
    """The form is fixed when a frame is enqueued: frame f is submitted while the tracker is alone, a companion is created,
    frame f+1 is submitted (single-role), and both are collected; later the same with the companion closed.  The frames
    equal the blocking calls of a lone tracker, and the last one enqueued ran the form of its enqueue."""
    frames = _frames(15, 16)
    gc.collect()
    a = _tracker(gf)
    want = []
    for t, g, d in frames:
        obs = a.trackImageRaw(t, g, d).copy()
        want.append((obs.tobytes(), a.last_status.copy(), dict(a.last_info)))
    a.close()
    b = _tracker(gf)
    companion = None
    got = []

    def collect():
        obs = b.wait().copy()
        got.append((obs.tobytes(), b.last_status.copy(), dict(b.last_info)))

    k = 0
    while k < len(frames):
        b.submit(*frames[k])
        if k in (4, 10):                     # switch between two submits
            if companion is None:
                companion = _tracker(gf)
            else:
                companion.close()
                companion = None
            b.submit(*frames[k + 1])
            collect()
            k += 1
        collect()
        check_form(k, b, "single-role" if companion is not None else "two-role")
        k += 1
    assert companion is None
    b.close()
    assert len(got) == len(want)
    for k, (x, y) in enumerate(zip(want, got)):
        assert x[2] == y[2], "frame %d: %s vs %s" % (k, x[2], y[2])
        assert np.array_equal(x[1], y[1]), "frame %d: status" % k
        assert x[0] == y[0], "frame %d: observations" % k


def test_group_beside_an_ungrouped_tracker(gf):
    """A TrackerGroup of two members and one ungrouped tracker on the same device: all three run the single-role form and
    match the oracle frame by frame."""
    from ground_fusion_b200.feature_tracker import TrackerGroup
    from oracle.fe_oracle import FeatureTrackerOracle
    gc.collect()
    mem = [_tracker(gf) for _ in range(2)]
    G = TrackerGroup(mem)
    lone = _tracker(gf)
    ref = [FeatureTrackerOracle(_cam(), 150, 30, 1, 1) for _ in range(3)]
    streams = [_frames(30 + i, 10) for i in range(3)]
    for k in range(10):
        fr = [s[k] for s in streams]
        G.submit([f[0] for f in fr[:2]], [f[1].ctypes.data for f in fr[:2]], [f[2].ctypes.data for f in fr[:2]])
        out = G.wait()
        got = lone.trackImageRaw(*fr[2])
        for i, tr in enumerate(mem + [lone]):
            want = ref[i].trackImage(*fr[i])
            check_oracle(k, tr, out[i][0] if i < 2 else got, ref[i], want)
            check_form(k, tr, "single-role")
    G.close()
    for tr in mem + [lone]:
        tr.close()


def _stripes(w, h):
    """Columns 0, 0, 255, 255 repeated, every 24th row 128; and the same shifted by half a period (two columns): every
    Scharr x-derivative of a full stripe row is +-4080 and every mismatch +-8160, and all the products of one pair chain
    (one column phase) have the same sign."""
    x = np.arange(w)
    a = np.tile(np.where(x % 4 < 2, 0, 255).astype(np.uint8), (h, 1))
    a[::24] = 128
    return a, np.ascontiguousarray(np.roll(a, 2, axis=1))


def b_partials(gx, gy, d):
    """[component][chain][positive, negative]: the per-chain sums lk_bpart_write accumulates in uint32 on the first
    iteration, from exact integer terms: pmaddwd pair units (columns k, k+4 | k+8, k+12) for chains 0..3, single pixels
    of columns 16..20 for the tail chain 4."""
    out = np.zeros((2, 5, 2), np.int64)
    for ci, g in enumerate((gx, gy)):
        t = d * g
        pair = t[:, 0:16].reshape(21, 2, 2, 4).sum(2)            # [row][half][k]: t[c] + t[c + 4], c = 8 * half + k
        units = [pair[:, :, k].ravel() for k in range(4)] + [t[:, 16:21].ravel()]
        for k, u in enumerate(units):
            out[ci, k] = u[u > 0].sum(), -u[u < 0].sum()
    return out


def test_largest_integer_partials(gf, lk_form):
    """Windows whose first-iteration b partials come as close to the bounds lk_bpart_write states as an 8-bit image allows
    (|d| <= 8160, |g| <= 4080, every chain below 2^32): a row of step edges under a shift of opposite sign.  The host computes
    the partials exactly and asserts how close they come; both forms must then match cv2 bit for bit (the partials exceed
    2^24, so the iteration takes the chain path, after summing them without wrapping)."""
    W, H = 640, 480
    a, b = _stripes(W, H)
    pts = np.array([(x, 24 * m + 10) for m in range(1, 19) for x in range(40, 600, 3)], np.float32)
    pair_max = 42 * 2 * 8160 * 4080          # 42 pair units of two products each
    tail_max = 105 * 8160 * 4080
    top = np.zeros(2, np.int64)
    for x, y in pts.astype(int):
        gx, gy, d = window_terms(a, b, x, y)
        assert np.abs(d).max() == 8160 and np.abs(gx).max() == 4080
        me, det = min_eig(gx, gy)
        assert me > 1e-2 and det > 1.0, (x, y, me, det)          # tracked, not rejected by minEig
        P = b_partials(gx, gy, d)
        assert P.max() < 1 << 32
        top = np.maximum(top, [P[:, :4].max(), P[:, 4].max()])
    assert top[0] >= 0.94 * pair_max and top[1] >= 0.56 * tail_max, (top / [pair_max, tail_max])
    for m in (0, 3):
        _, st = check_lk(gf, a, b, pts, m, lk_form)
        assert st.all()
