"""GPU parity tests of the front end away from its usual operating point (run with -m gpu on an H100).

test_fe_gpu.py checks the front end mostly at 640x480 with small motion, where every pyramid level is at least 80 px wide
and the LK windows are staged by 2-D TMA.  This module covers the other geometries and code paths, bit-exact against
cv2 4.13 (stage entry points) or oracle/fe_oracle.py (tracker):
  - LK in both of its forms (two warp roles, a tracker alone on its device; single role, several trackers) with the TMA
    staging on and off (GF_LK_NO_TMA, and images below 640 px wide, where it is off for the whole tracker), widths that are not multiples of 16, portrait images, 1080p, large motion that restages the search window,
    windows on the image border at every level, flat and clipped textures, initial flow far from the truth;
  - cornerMinEigenVal at widths that are not multiples of 32;
  - goodFeaturesToTrack with more than 65536 candidates, a grown min-distance cell and an overflowing mask tile;
  - tracker sequences at those geometries, from row-padded frames, and with every orchestration switch;
  - the solver with programmatic dependent launch off.
Each test that targets a path also asserts, from values computed on the host, that its input reaches that path.
"""
import math
import os
import subprocess
import sys

import numpy as np
import pytest

from conftest import make_texture_image, warp_image
from test_fe_gpu import _padded, _run_sequence, lk_form, lk_staging  # noqa: F401 (fixtures)

pytestmark = pytest.mark.gpu
cv2 = pytest.importorskip("cv2")

TESTS = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(TESTS)
CRIT = (cv2.TERM_CRITERIA_COUNT + cv2.TERM_CRITERIA_EPS, 30, 0.01)    # cv2's default, and the library's
LK_SHAPES = [(640, 480), (641, 481), (752, 480), (480, 640), (1280, 720), (1920, 1080), (424, 400)]


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def level_sizes(w, h, n=4):
    out = [(w, h)]
    for _ in range(n - 1):
        w, h = (w + 1) // 2, (h + 1) // 2
        out.append((w, h))
    return out


def lk_levels(w, h):
    """max_level values gf_stage_lk accepts: the coarsest level at least 48x48."""
    return [m for m in range(4) if (w >> m) >= 48 and (h >> m) >= 48]


def lk_tma_on(w, h, max_level):
    """Mirror of make_lk_maps (fe_tracker.cu): TMA staging needs every level used at least 80 px wide and 40 px high."""
    if os.environ.get("GF_LK_NO_TMA"):
        return False
    return all(lw >= 80 and lh >= 40 for lw, lh in level_sizes(w, h)[:max_level + 1])


def nms_cell_size(w, h, min_dist):
    """Mirror of alloc_nms_grid (fe_tracker.cu): cell of at least max(min_dist, 16), grown until the grid fits 160 KB."""
    cs = max(min_dist, 16)
    while (-(-w // cs) + 2) * (-(-h // cs) + 2) * 32 > 160 * 1024:
        cs += 1
    return cs


def max_tile_apron(kept, w, h, r):
    """Most kept features any 64x16 mask tile collects (mask_tile_load, fe_select.cuh: rounded centres within r of it)."""
    c = np.rint(np.asarray(kept, np.float32)).astype(np.int64).reshape(-1, 2)
    best = 0
    for y0 in range(0, h, 16):
        for x0 in range(0, w, 64):
            m = (c[:, 0] >= x0 - r) & (c[:, 0] < x0 + 64 + r) & (c[:, 1] >= y0 - r) & (c[:, 1] < y0 + 16 + r)
            best = max(best, int(m.sum()))
    return best


def check_lk(gf, a, b, pts, max_level, form, init=None):
    """gf_stage_lk in the LK form `form` (the lk_form fixture's value) against cv2.calcOpticalFlowPyrLK, bit for bit; returns
    cv2's (points, status)."""
    pts = np.ascontiguousarray(pts, np.float32).reshape(-1, 2)
    nxt = None if init is None else np.ascontiguousarray(init, np.float32).reshape(-1, 1, 2).copy()
    flags = 0 if init is None else cv2.OPTFLOW_USE_INITIAL_FLOW
    q_cv, st_cv, _ = cv2.calcOpticalFlowPyrLK(a, b, pts.reshape(-1, 1, 2), nxt, winSize=(21, 21), maxLevel=max_level,
                                              criteria=CRIT, flags=flags)
    q_cv, st_cv = q_cv.reshape(-1, 2), st_cv.ravel()
    q, st = gf.calc_optical_flow_pyr_lk(a, b, pts, max_level, init=init, roles=form == "two-role")
    bad = np.flatnonzero((st != st_cv) | np.any(bits(q) != bits(q_cv), 1))
    if len(bad):
        i = bad[0]
        pytest.fail("%s: %d of %d points differ; first: p=%r gpu %r/%d cv2 %r/%d" % (form, len(bad), len(pts), tuple(pts[i]),
                                                                                   tuple(q[i]), st[i], tuple(q_cv[i]), st_cv[i]))
    return q_cv, st_cv


def boundary_points(w, h, max_level):
    """Points whose window origin floor(p/2^l - 10) is -22, -21, -20, w_l-25, w_l-24, w_l-1 or w_l (same in y) at each level
    l <= max_level, at integer and .5 coordinates, in every combination with each other and with the centre, plus points
    far outside the image."""
    out = []
    for l, (lw, lh) in enumerate(level_sizes(w, h)[:max_level + 1]):
        s = float(1 << l)
        kx = [-22, -21, -20, lw - 25, lw - 24, lw - 1, lw, lw // 2 - 10]
        ky = [-22, -21, -20, lh - 25, lh - 24, lh - 1, lh, lh // 2 - 10]
        for f in (0.0, 0.5):
            for x in kx:
                for y in ky:
                    out.append(((x + 10 + f) * s, (y + 10 + f) * s))
    out += [(-100, h / 2), (w + 100, h / 2), (w / 2, -100), (w / 2, h + 100), (-1000, -1000), (w + 1000, h + 1000), (-30.5, -30.5)]
    p = np.array(out, np.float32)
    for l, (lw, lh) in enumerate(level_sizes(w, h)[:max_level + 1]):      # the construction is exact in float32
        o = np.floor(p * np.float32(1.0 / (1 << l)) - np.float32(10)).astype(np.int64)
        assert {-22, -21, -20, lw - 25, lw - 24, lw - 1, lw} <= set(o[:, 0].tolist())
        assert {-22, -21, -20, lh - 25, lh - 24, lh - 1, lh} <= set(o[:, 1].tolist())
    return p


# ---- A. LK ------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("w,h", LK_SHAPES)
def test_lk_geometries_and_border_windows(gf, lk_form, lk_staging, w, h):
    """Every accepted max_level at each shape, TMA staging on and off: random points (some just outside the image) and the
    constructed border points of every level, small motion with rotation."""
    if (w, h) == (424, 400):
        assert level_sizes(w, h)[3][0] < 80 and not lk_tma_on(w, h, 3)       # below 640 px wide the staging is per-thread
    seed = w + h
    a = make_texture_image(seed, w, h, contrast=1.5)
    b = warp_image(a, 3.3, -2.1, 0.7)
    rng = np.random.default_rng(seed)
    rand = np.stack([rng.uniform(-5, w + 5, 400), rng.uniform(-5, h + 5, 400)], 1).astype(np.float32)
    levels = lk_levels(w, h)
    assert levels == [0, 1, 2, 3]
    for m in levels:
        pts = np.concatenate([rand, boundary_points(w, h, m)])
        check_lk(gf, a, b, pts, m, lk_form)


def _lk_iterates(a, b, pts):
    """cv2's level-0 iterates: Q[k] is the point after k iterations (Q[0] = pts), k = 0..30."""
    Q = [pts.astype(np.float32)]
    for k in range(1, 31):
        q, _, _ = cv2.calcOpticalFlowPyrLK(a, b, pts.reshape(-1, 1, 2), None, winSize=(21, 21), maxLevel=0,
                                           criteria=(cv2.TERM_CRITERIA_COUNT + cv2.TERM_CRITERIA_EPS, k, 0.01))
        Q.append(q.reshape(-1, 2))
    return Q


def restaged_windows(a, b, pts):
    """Replays lk_level's search-window logic (fe_lk.cuh) on cv2's iterates at max_level 0: the 40x40 window starts at
    floor(p - 10) - 9 and is restaged when an iterate's 22x22 read leaves it.  Returns (restaged, restaged onto the border
    from a window inside the image), per point."""
    h, w = a.shape
    Q = _lk_iterates(a, b, pts)
    win = np.floor(pts - 10).astype(np.int64) - 9

    def inside(o):
        return (o[:, 0] >= 0) & (o[:, 1] >= 0) & (o[:, 0] + 40 <= w) & (o[:, 1] + 40 <= h)

    start_inside = inside(win)
    restaged = np.zeros(len(pts), bool)
    to_border = np.zeros(len(pts), bool)
    for k in range(1, 30):
        ran = np.any(Q[k + 1] != Q[k], 1)                  # iteration k+1 read the window at Q[k]
        iq = np.floor(Q[k] - 10).astype(np.int64)
        in_range = (iq[:, 0] >= -21) & (iq[:, 0] < w) & (iq[:, 1] >= -21) & (iq[:, 1] < h)
        leaves = np.any((iq < win) | (iq + 22 > win + 40), 1)
        re = ran & in_range & leaves
        win[re] = iq[re] - 9
        restaged |= re
        to_border |= re & start_inside & ~inside(win)
    return restaged, to_border


def _band_points(rng, w, h, n):
    """Points 22-60 px inside each image edge: their search windows start inside the image and can move onto the border."""
    d = rng.uniform(22, 60, n)
    side = rng.integers(0, 4, n)
    x = np.where(side == 0, d, np.where(side == 1, w - d, rng.uniform(0, w, n)))
    y = np.where(side == 2, d, np.where(side == 3, h - d, rng.uniform(0, h, n)))
    return np.stack([x, y], 1).astype(np.float32)


@pytest.mark.parametrize("w,h", [(640, 480), (641, 481), (424, 400), (1280, 720)])
@pytest.mark.parametrize("max_level,dx,dy,ang", [(0, 13.4, -12.2, 0.0), (0, 24.7, 18.1, 1.0), (1, 29.3, -21.6, 1.5),
                                                 (3, 47.5, 31.2, 2.0), (3, -86.3, 44.9, -4.0)])
def test_lk_large_motion(gf, lk_form, lk_staging, w, h, max_level, dx, dy, ang):
    """Shifts of 12-30 px at max_level 0 and 1, 40-90 px with rotation at max_level 3: the search window is restaged during
    the iterations, from the interior onto the border among others.  A coarser texture widens the basin of convergence."""
    seed = 7 * w + max_level
    a = make_texture_image(seed, w, h, sigma=6.0, contrast=2.0)
    b = warp_image(a, dx, dy, ang)
    rng = np.random.default_rng(seed)
    pts = np.concatenate([np.stack([rng.uniform(0, w, 400), rng.uniform(0, h, 400)], 1).astype(np.float32),
                          _band_points(rng, w, h, 200)])
    check_lk(gf, a, b, pts, max_level, lk_form)
    if max_level == 0:
        restaged, to_border = restaged_windows(a, b, pts)
        assert restaged.sum() >= 50, "only %d points restage their search window" % restaged.sum()
        assert to_border.sum() >= 5, "only %d search windows move from the interior onto the border" % to_border.sum()


def _constant_windows(img, pts, max_level):
    """[n, max_level+1]: the 24x24 template window of the point at that level lies inside the level and is constant
    (zero gradient matrix: the minimum-eigenvalue test rejects it)."""
    pyr = [img]
    for _ in range(max_level):
        pyr.append(cv2.pyrDown(pyr[-1]))
    out = np.zeros((len(pts), max_level + 1), bool)
    for l, L in enumerate(pyr):
        lh, lw = L.shape
        o = np.floor(pts * np.float32(1.0 / (1 << l)) - np.float32(10)).astype(np.int64) - 1
        for i, (x, y) in enumerate(o):
            if x >= 0 and y >= 0 and x + 24 <= lw and y + 24 <= lh:
                win = L[y:y + 24, x:x + 24]
                out[i, l] = win.min() == win.max()
    return out


@pytest.mark.parametrize("w,h", [(640, 480), (641, 481), (424, 400)])
def test_lk_flat_and_clipped_texture(gf, lk_form, lk_staging, w, h):
    """A tone curve clips a coarse texture to 0 and 255 over large areas, and a block is constant at 7: the minimum-eigenvalue
    rejection fires at coarse levels (the point continues with twice the guess) and at level 0 (status 0)."""
    t = make_texture_image(w + 3 * h, w, h, sigma=8.0, contrast=1.0).astype(np.float32)
    a = np.clip((t - 128.0) * 4.0 + 128.0, 0, 255).astype(np.uint8)
    a[h // 3:h // 3 + 200, w // 4:w // 4 + 200] = 7
    b = warp_image(a, 2.6, 1.9, 0.5)
    rng = np.random.default_rng(w)
    pts = np.concatenate([np.stack([rng.uniform(0, w, 500), rng.uniform(0, h, 500)], 1),
                          np.stack([rng.uniform(w // 4, w // 4 + 200, 60), rng.uniform(h // 3, h // 3 + 200, 60)], 1)]).astype(np.float32)
    for m in lk_levels(w, h):
        _, st = check_lk(gf, a, b, pts, m, lk_form)
        flat = _constant_windows(a, pts, m)
        assert np.any(flat[:, 0] & (st == 0)), "no level-0 rejection"
        if m > 0:
            assert flat[:, 1:].any(), "no coarse-level rejection"


@pytest.mark.parametrize("w,h", [(641, 481), (480, 640)])
@pytest.mark.parametrize("max_level", [1, 3])
def test_lk_initial_flow_far_from_truth(gf, lk_form, lk_staging, w, h, max_level):
    a = make_texture_image(w + 2 * h, w, h, sigma=4.0, contrast=1.5)
    b = warp_image(a, 2.2, -1.6, 0.3)
    rng = np.random.default_rng(h)
    pts = np.stack([rng.uniform(-5, w + 5, 500), rng.uniform(-5, h + 5, 500)], 1).astype(np.float32)
    init = pts + np.stack([rng.uniform(-14, 14, 500), rng.uniform(-14, 14, 500)], 1).astype(np.float32)
    check_lk(gf, a, b, pts, max_level, lk_form, init=init)


# ---- B. cornerMinEigenVal and goodFeaturesToTrack ---------------------------------------------------------------------

@pytest.mark.parametrize("w", [377, 383, 400, 511, 513, 641, 650, 752, 1920])
@pytest.mark.parametrize("odd_h", [False, True])
def test_min_eig_widths(gf, w, odd_h):
    h = (w * 3 // 4) | 1 if odd_h else (w * 3 // 4) & ~1
    img = make_texture_image(w + h, w, h, contrast=1.8)
    img[: h // 5, : w // 6] = 255                            # a flat corner block at the border
    e, _ = gf.corner_min_eigen_val(img)
    want = cv2.cornerMinEigenVal(img, 3, ksize=3)
    assert np.array_equal(bits(e), bits(want)), "%d px differ" % (bits(e) != bits(want)).sum()


def check_gftt(gf, img, max_corners, min_dist, kept):
    assert len(kept) + max_corners <= 1024
    mask = np.full(img.shape, 255, np.uint8)
    for p in kept:
        cv2.circle(mask, (int(np.rint(p[0])), int(np.rint(p[1]))), min_dist, 0, -1)
    want = cv2.goodFeaturesToTrack(img, max_corners, 0.01, min_dist, mask=mask)
    want = np.zeros((0, 2), np.float32) if want is None else want.reshape(-1, 2)
    got, info = gf.good_features_to_track(img, max_corners, min_dist, kept)
    assert got.shape == want.shape and np.array_equal(got, want), info
    return info


@pytest.mark.parametrize("w,h", LK_SHAPES)
@pytest.mark.parametrize("min_dist", [5, 7, 20, 30])
def test_gftt_geometries(gf, w, h, min_dist):
    img = make_texture_image(w * 7 + min_dist, w, h, contrast=1.3)
    rng = np.random.default_rng(min_dist)
    kept = np.stack([rng.uniform(1, w - 2, 100), rng.uniform(1, h - 2, 100)], 1).astype(np.float32)
    check_gftt(gf, img, 600, min_dist, kept)


@pytest.mark.parametrize("min_dist,n_kept", [(5, 0), (7, 200), (20, 0)])
def test_gftt_1080p_slow_paths(gf, min_dist, n_kept):
    """More than NMS_MAX_PER_THREAD x 1024 = 65536 candidates (liveness of the rest in HBM) and a cell grid grown past
    max(min_dist, 16) to fit shared memory."""
    w, h = 1920, 1080
    img = make_texture_image(min_dist, w, h)
    rng = np.random.default_rng(min_dist)
    kept = np.stack([rng.uniform(1, w - 2, n_kept), rng.uniform(1, h - 2, n_kept)], 1).astype(np.float32)
    info = check_gftt(gf, img, 1024 - n_kept, min_dist, kept)
    assert info["n_candidates"] > 65536, info
    assert nms_cell_size(w, h, min_dist) > max(min_dist, 16)


def _hex_lattice(x0, y0, x1, y1, dx, dy):
    pts = []
    for k, y in enumerate(range(y0, y1, dy)):
        pts += [(x, y) for x in range(x0 + (k % 2) * (dx // 2), x1, dx)]
    return np.array(pts, np.float32) + np.float32(0.25)


@pytest.mark.parametrize("w,h", [(640, 480), (641, 481)])
def test_gftt_dense_kept_overflows_mask_tile(gf, w, h):
    """Kept features more than min_dist apart, packed on a lattice: more than MASK_LIST = 64 of them reach one tile's apron,
    so the masked maximum and the candidates take the exact slow path of mask_open (fe_select.cuh)."""
    r = 5
    kept = _hex_lattice(90, 100, 300, 190, 6, 5)
    c = np.rint(kept).astype(np.int64)
    d2 = ((c[:, None, :] - c[None, :, :]) ** 2).sum(-1)
    assert (d2[~np.eye(len(c), dtype=bool)] > r * r).all()      # every pair more than r apart
    assert max_tile_apron(kept, w, h, r) > 64
    img = make_texture_image(w, w, h, contrast=1.2)
    check_gftt(gf, img, 1024 - len(kept), r, kept)


# ---- C. tracker sequences ---------------------------------------------------------------------------------------------

def test_track_sequence_424x400_without_tma(gf, lk_form):
    assert level_sizes(424, 400)[3][0] < 80 and not lk_tma_on(424, 400, 3)
    _run_sequence(gf, seed=3, n_frames=20, w=424, h=400, max_cnt=150, min_dist=20, form=lk_form)


def test_track_sequence_641x481_padded_rows(gf, lk_form):
    _run_sequence(gf, seed=4, n_frames=20, w=641, h=481, max_cnt=200, min_dist=25, pad=23, form=lk_form)


def test_track_sequence_480x640_portrait(gf, lk_form):
    """The reference reads the saturation test as at<uchar>((int)x, (int)y): row x, column y.  In a portrait image that read
    is in bounds for every point with x < 640 and y < 480, i.e. most of them.  The camera is IDC_CAM turned by 90 degrees
    (the landscape intrinsics would put the bottom rows where the radial model diverges)."""
    from oracle.fe_oracle import IDC_CAM as C, PinholeCamera
    cam = PinholeCamera(C["fy"], C["fx"], C["cy"], C["cx"], C["k1"], C["k2"], C["p2"], C["p1"])
    seen = []
    _run_sequence(gf, seed=5, n_frames=20, w=480, h=640, max_cnt=150, min_dist=25, cam=cam, form=lk_form,
                  on_frame=lambda k, g, ref, got: seen.append(int(((got["v"][:, 3] < 640) & (got["v"][:, 4] < 480)).sum())))
    assert sum(seen) > 1000


def test_track_sequence_752x480(gf, lk_form):
    _run_sequence(gf, seed=6, n_frames=20, w=752, h=480, max_cnt=150, min_dist=30, form=lk_form)


def test_track_sequence_1080p_gftt_slow_paths(gf, lk_form):
    """150 features at 1920x1080, min_dist 20: more than 65536 candidates and a grown cell grid inside the tracker."""
    assert nms_cell_size(1920, 1080, 20) > 20
    cands = []
    _run_sequence(gf, seed=7, n_frames=10, w=1920, h=1080, max_cnt=150, min_dist=20, form=lk_form,
                  on_frame=lambda k, g, ref, got: cands.append(g.last_info["n_candidates"]))
    assert max(cands) > 65536, cands


def test_track_sequence_dense_1000_features(gf, lk_form):
    """max_cnt 1000 at min_dist 5: setMask's std::sort replay and the disk tests near capacity."""
    aprons = []

    def on_frame(k, g, ref, got):
        nk = len(ref.ids) - len(ref.last_n_pts)
        aprons.append(max_tile_apron(ref.prev_pts[:nk], 640, 480, 5) if nk else 0)
        assert len(got) > 900

    _run_sequence(gf, seed=8, n_frames=12, max_cnt=1000, min_dist=5, on_frame=on_frame, form=lk_form)
    assert max(aprons) > 8


def _frame_ptrs(frames, on_device, pad, keep):
    """Frame addresses for trackBatch: host frames as views into rows `pad` elements wider, or packed device copies."""
    import torch
    if on_device:
        gs = [torch.from_numpy(np.ascontiguousarray(g)).cuda() for _, g, _ in frames]
        ds = [(torch.from_numpy(np.ascontiguousarray(d).view(np.int16)).cuda() if d is not None else None) for _, _, d in frames]
        keep.append((gs, ds))
        torch.cuda.synchronize()
        return [x.data_ptr() for x in gs], [(x.data_ptr() if x is not None else 0) for x in ds], None, None
    gs = [_padded(g, pad) for _, g, _ in frames]
    ds = [(_padded(d, pad) if d is not None else None) for _, _, d in frames]
    keep.append((gs, ds))
    return ([g.ctypes.data for g in gs], [(d.ctypes.data if d is not None else 0) for d in ds], gs[0].strides[0],
            next(d.strides[0] for d in ds if d is not None))


def _check_frames(want, got, base=0):
    assert len(want) == len(got)
    for k, ((o1, s1, i1), (o2, s2, i2)) in enumerate(zip(want, got)):
        assert i1 == i2, "frame %d: %s vs %s" % (base + k, i1, i2)
        assert np.array_equal(s1, s2), "frame %d" % (base + k)
        assert o1.tobytes() == o2.tobytes(), "frame %d" % (base + k)


@pytest.mark.parametrize("w,h", [(641, 481), (424, 400), (752, 480), (480, 640)])
@pytest.mark.parametrize("on_device", [False, True])
def test_batch_odd_geometry_equals_track_image(gf, w, h, on_device):
    """trackBatch at widths whose rows are not 16-byte aligned, at 752x480 and in portrait, host frames with a row pitch
    larger than the width, frames without a depth image in between; compared with trackImage."""
    from ground_fusion_b200.synth import SyntheticStream
    from oracle.fe_oracle import IDC_CAM, PinholeCamera
    sc = w / 640.0
    cam = PinholeCamera(IDC_CAM["fx"] * sc, IDC_CAM["fy"] * sc, IDC_CAM["cx"] * sc, IDC_CAM["cy"] * sc,
                        IDC_CAM["k1"], IDC_CAM["k2"], IDC_CAM["p1"], IDC_CAM["p2"])
    stream = SyntheticStream(seed=12, width=w, height=h)
    frames = [stream.frame(k) for k in range(13)]
    frames = [(t, g, (d if k % 5 != 3 else None)) for k, (t, g, d) in enumerate(frames)]
    a = gf.FeatureTracker(w, h, cam.params8(), 150, 25, 1, 1)
    b = gf.FeatureTracker(w, h, cam.params8(), 150, 25, 1, 1)
    keep = []
    pos = 0
    for n in (1, 5, 7):
        fr = frames[pos:pos + n]
        want = []
        for t, g, d in fr:
            obs = a.trackImageRaw(t, g, d).copy()
            want.append((obs, a.last_status.copy(), dict(a.last_info)))
        gp, dp, gpitch, dpitch = _frame_ptrs(fr, on_device, 19, keep)
        got = b.trackBatch([t for t, _, _ in fr], gp, dp, on_device=on_device, gray_pitch=gpitch, depth_pitch=dpitch)
        _check_frames(want, got, pos)
        pos += n
    assert sum(len(o) for o, _, _ in got) > 500
    a.close(); b.close()


# ---- D. orchestration switches ----------------------------------------------------------------------------------------

@pytest.mark.parametrize("switch", ["GF_NO_GRAPH", "GF_LK_NO_TMA"])
@pytest.mark.parametrize("on_device", [False, True])
def test_tracker_switch_matches_oracle(gf, monkeypatch, switch, on_device):
    """Each documented switch (read when the tracker is created): a 20-frame C2 sequence against the oracle, then the same
    frames through trackBatch, from host or device memory."""
    from ground_fusion_b200.synth import SyntheticStream
    from oracle.fe_oracle import IDC_CAM, PinholeCamera
    monkeypatch.setenv(switch, "1")
    want = []
    _run_sequence(gf, seed=0, n_frames=20,
                  on_frame=lambda k, g, ref, got: want.append((got.copy(), g.last_status.copy(), dict(g.last_info))))
    cam = PinholeCamera(**IDC_CAM)
    stream = SyntheticStream(seed=0)
    frames = [stream.frame(k) for k in range(20)]
    keep = []
    gp, dp, gpitch, dpitch = _frame_ptrs(frames, on_device, 0, keep)
    b = gf.FeatureTracker(640, 480, cam.params8(), 150, 30, 1, 1)
    got = b.trackBatch([t for t, _, _ in frames], gp, dp, on_device=on_device, gray_pitch=gpitch, depth_pitch=dpitch)
    _check_frames(want, got)
    b.close()


def test_ba_solve_without_pdl_matches_oracle():
    """GF_BA_NO_PDL is read once per process: one C2 solve (max_iter 8) in a fresh interpreter with it set, to the bar of
    test_ba_gpu.py."""
    code = "\n".join([
        "import sys",
        "sys.path[:0] = [%r, %r]" % (ROOT, TESTS),
        "from test_ba_gpu import compare",
        "from ground_fusion_b200.estimator import BundleAdjuster",
        "from ground_fusion_b200.synth_ba import make_window",
        "ba = BundleAdjuster(0)",
        "pb, _ = make_window(seed=0)",
        "s = compare(ba, pb, 8)",
        "ba.close()",
        "print('solved', s['reduced_dim'], s['iterations'])",
    ])
    flags = [f for f, on in (("-s", sys.flags.no_user_site), ("-E", sys.flags.ignore_environment)) if on]
    env = dict(os.environ, GF_BA_NO_PDL="1")
    r = subprocess.run([sys.executable] + flags + ["-c", code], env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "solved 165 " in r.stdout, r.stdout
