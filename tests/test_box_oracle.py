"""CPU: trackImagebox's box test pinned to cv2, the oracle's trackImagebox, the default synthetic stream, the adaptor's build.

The device code does not run a polygon test: it evaluates the closed form of box_ref.closed_form, and these tests are what
make that legitimate -- it equals `cv2.pointPolygonTest(contour, pt, true) > 0` (cv2 4.13) on every probe, including the int64 ->
int wrap of the message fields and corners beyond 2^24, where int -> float rounding merges neighbouring corners."""
import os
import subprocess

import numpy as np
import pytest

from box_ref import FeatureTrackerOracleBox, FeatureTrackerOracleFastBox, closed_form, cv2_inside, probe_sets, wrap32

cv2 = pytest.importorskip("cv2")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_closed_form_equals_point_polygon_test():
    n = inside = 0
    for box, pts in probe_sets(seed=0):
        want = np.array([cv2_inside(box, p) for p in pts])
        assert np.array_equal(closed_form([box], pts), want), box
        n += len(pts); inside += int(want.sum())
    assert n > 150000 and 0.1 * n < inside < 0.5 * n, (n, inside)


def test_probe_sets_reach_the_edge_cases():
    """The probes include what makes the closed form non-obvious: a wrap of int64 fields, corners whose int -> float conversion
    rounds, and the strict boundary (points one ulp inside and on the edge)."""
    sets = probe_sets(seed=0)
    wrapped = sum(any(wrap32(v) != v for v in b) for b, _ in sets)
    rounded = sum(any(float(np.float32(wrap32(v))) != wrap32(v) for v in b) for b, _ in sets)
    assert wrapped > 200 and rounded > 500, (wrapped, rounded)
    b = np.array([10, 20, 30, 40], np.int64)
    pts = np.array([[10, 30], [np.nextafter(np.float32(10), np.float32(11)), 30], [20, 40], [20, np.nextafter(np.float32(40), np.float32(0))]],
                   np.float32)
    assert closed_form([b], pts).tolist() == [False, True, False, True]
    assert [cv2_inside(b, p) for p in pts] == [False, True, False, True]
    assert not closed_form([np.array([5, 5, 5, 50])], [[5, 20]])[0] and not cv2_inside([5, 5, 5, 50], (5, 20))
    assert closed_form([np.array([30, 40, 10, 20])], [[20, 30]])[0] and cv2_inside([30, 40, 10, 20], (20, 30))     # inverted


def test_closed_form_over_many_boxes():
    """A feature is left out when it is inside ANY box: up to 100 boxes per frame (darknet_ros's limit)."""
    rng = np.random.default_rng(1)
    for nb in (1, 7, 100):
        boxes = [np.sort(rng.integers(0, 640, 2)).tolist() + [0, 0] for _ in range(nb)]
        boxes = np.array([[b[0], y, b[1], y + int(rng.integers(0, 120))] for b, y in zip(boxes, rng.integers(0, 400, nb))], np.int64)
        pts = np.stack([rng.uniform(0, 640, 3000), rng.uniform(0, 480, 3000)], 1).astype(np.float32)
        want = np.array([any(cv2_inside(b, p) for b in boxes) for p in pts])
        assert np.array_equal(closed_form(boxes, pts), want) and want.any()


def _cam():
    from oracle.fe_oracle import IDC_CAM, PinholeCamera
    return PinholeCamera(**IDC_CAM)


@pytest.mark.parametrize("cls", [FeatureTrackerOracleBox, FeatureTrackerOracleFastBox])
@pytest.mark.parametrize("depth_cam", [1, 0])
def test_oracle_trackimagebox_is_trackimage_minus_the_box_filter(cls, depth_cam):
    """trackImagebox leaves exactly the boxed features out of trackImage's frame and changes nothing else: a second oracle fed no
    boxes ends every frame in the same state (ids, points, track counts)."""
    from ground_fusion_b200.synth import SyntheticStream
    from oracle.fe_oracle import FeatureTrackerOracle
    st = SyntheticStream(seed=0, dynamic=True)
    a, b = cls(_cam(), 150, 30, 1, depth_cam), FeatureTrackerOracle(_cam(), 150, 30, 1, depth_cam)
    dropped = 0
    for k in range(8):
        t, g, d = st.frame(k)
        boxes = st.boxes(k) if k % 3 != 2 else np.array([[0, 0, 639, 479]], np.int64)
        got, full = a.trackImagebox(t, boxes, g, d), b.trackImage(t, g, d)
        assert list(a.ids) == list(b.ids) and np.array_equal(a.cur_pts, b.cur_pts) and list(a.track_cnt) == list(b.track_cnt)
        pts = np.array([full[i][3:5] for i in full], np.float32)
        inside = closed_form(boxes, pts)
        assert sorted(got) == sorted(np.array(list(full))[~inside].tolist())
        for fid in got:
            assert np.array_equal(got[fid], full[fid])
        if k % 3 == 2:
            assert got == {}                             # a box over the whole image: nothing reaches the estimator
        dropped += int(inside.sum())
    assert dropped > 150, dropped


def test_default_synthetic_stream_is_unchanged():
    """The moving object is off by default: the oracle on the default stream still reproduces the committed fixture, and the
    dynamic stream differs from it only inside the object's box, where the object is nearer than the plane."""
    from ground_fusion_b200.synth import SyntheticStream
    from oracle.fe_oracle import FeatureTrackerOracle
    g = np.load(os.path.join(ROOT, "tests", "golden", "fe_c2_seed0.npz"))
    seed, w, h, max_cnt, min_dist = (int(v) for v in g["meta"][:5])
    st = SyntheticStream(seed=seed, width=w, height=h)
    ref = FeatureTrackerOracle(_cam(), max_cnt, min_dist, 1, 1)
    for k in range(3):
        t, gray, depth = st.frame(k)
        want = ref.trackImage(t, gray, depth)
        assert np.array_equal(np.array(ref.ids), g["ids_%d" % k])
        assert np.array_equal(np.array([want[i] for i in ref.ids]), g["obs_%d" % k])
        assert len(st.boxes(k)) == 0
    _, gray, depth = st.frame(0)
    dyn = SyntheticStream(seed=seed, width=w, height=h, dynamic=True)
    _, g2, d2 = dyn.frame(0)
    (x0, y0, x1, y1), = dyn.boxes(0)
    diff = np.argwhere(g2 != gray)
    assert len(diff) > 10000 and d2.min() < depth.min()
    assert x0 <= diff[:, 1].min() and diff[:, 1].max() <= x1 + 1 and y0 <= diff[:, 0].min() and diff[:, 0].max() <= y1 + 1


def test_adaptor_builds_with_trackimagebox():
    subprocess.check_call(["make", "-s", "-C", os.path.join(ROOT, "adaptor")])
    syms = subprocess.check_output(["nm", "-D", "--undefined-only", os.path.join(ROOT, "adaptor", "_build", "harness")]).decode()
    assert "gf_tracker_track" in syms.split()
