"""GPU tests of LK's level-by-level edge cases (run with -m gpu on an H100).

Each test runs in both LK forms (DESIGN.md §1.3) with the TMA staging on and off (GF_LK_NO_TMA), bit-exact against
cv2.calcOpticalFlowPyrLK (stage entry) or oracle/fe_oracle.py (tracker).  In the two-role form (fe_lk.cuh) consumer warps
iterate pyramid level l while producer warps build level l-1, and these cases drive the hand-over between the roles; the
single-role form (fe_lk_single.cuh) sets up and iterates each level with all warps, and they are its level edge cases too:
  - coarse levels rejected by minEig above a valid finest level;
  - levels that converge in one iteration (in the two-role form the consumers wait for the producers at every level);
  - the sequential-chain fallback on a coarse level;
  - max_level 0, a single level.
The host recomputes, exactly in integers, what each test needs its input to reach, and asserts it.
"""
import cv2
import numpy as np
import pytest

from conftest import make_texture_image, warp_image
from test_fe_edges_gpu import boundary_points, check_lk
from test_fe_gpu import _run_sequence, lk_debug, lk_form, lk_staging  # noqa: F401 (fixtures)

pytestmark = pytest.mark.gpu

W, H = 640, 480
FLT_SCALE = 1.0 / (1 << 20)


def pyramid(img, n=4):
    out = [img]
    for _ in range(n - 1):
        out.append(cv2.pyrDown(out[-1]))
    return out


def window_terms(I, J, x, y):
    """For integer level coordinates (x, y): the template values, Scharr derivatives and mismatch of LK's first iteration
    with the search window at the same place.  With integer coordinates every bilinear weight but the first is 0, so the
    fixed-point values are exact: the patch is 32 * I, the gradients the Scharr values, the mismatch 32 * (J - I)."""
    ix = cv2.Scharr(I, cv2.CV_16S, 1, 0).astype(np.int64)
    iy = cv2.Scharr(I, cv2.CV_16S, 0, 1).astype(np.int64)
    sl = (slice(y - 10, y + 11), slice(x - 10, x + 11))
    d = 32 * (J[sl].astype(np.int64) - I[sl].astype(np.int64))
    return ix[sl], iy[sl], d


def min_eig(gx, gy):
    """OpenCV's minEig and determinant of the level's gradient matrix (float64; the tests keep clear of the thresholds)."""
    a11, a12, a22 = (gx * gx).sum() * FLT_SCALE, (gx * gy).sum() * FLT_SCALE, (gy * gy).sum() * FLT_SCALE
    return (a22 + a11 - np.sqrt((a11 - a22) ** 2 + 4 * a12 * a12)) / (2 * 21 * 21), a11 * a22 - a12 * a12


def b_chains_exact(gx, gy, d):
    """Whether every b chain of the iteration is within the 2^24 bound of the integer shortcut (fe_lk.cuh): pmaddwd pair
    units (columns k, k+4 | k+8, k+12) for chains 0..3, single pixels of columns 16..20 for the tail chain."""
    for g in (gx, gy):
        t = d * g
        units = [[] for _ in range(5)]
        for r in range(21):
            for hh in range(2):
                for k in range(4):
                    c = 8 * hh + k
                    units[k].append(t[r, c] + t[r, c + 4])
            units[4].extend(t[r, 16:21].tolist())
        for u in units:
            u = np.array(u, np.int64)
            if u[u > 0].sum() >= 1 << 24 or -u[u < 0].sum() >= 1 << 24:
                return False
    return True


def test_coarse_levels_rejected_by_min_eig(gf, lk_form, lk_staging):
    """A texture of 2 x 2 px cells: pyrDown turns it into a one-pixel alternation at level 1, whose Scharr derivatives
    are all 0, and into near-flat grey above.  Levels 3..1 are built as rejected, level 0 is tracked."""
    yy, xx = np.mgrid[0:H, 0:W]
    checker = (((xx >> 1) + (yy >> 1)) & 1).astype(np.float32)
    a = np.clip(128 + 80 * (checker - 0.5) * (1 + 0.1 * np.sin(xx / 7.0) * np.cos(yy / 5.0)), 0, 255).astype(np.uint8)
    b = warp_image(a, 0.6, -0.4)
    pts = np.array([(x, y) for y in range(96, H - 96, 40) for x in range(96, W - 96, 40)], np.float32)
    PI, PJ = pyramid(a), pyramid(b)
    for x, y in pts.astype(int):
        for l in range(4):
            gx, gy, _ = window_terms(PI[l], PJ[l], x >> l, y >> l)
            me, _ = min_eig(gx, gy)
            assert (me > 2e-4) if l == 0 else (me < 5e-5), (x, y, l, me)
    _, st = check_lk(gf, a, b, pts, 3, lk_form)
    assert st.all()


def test_levels_converging_in_one_iteration(gf, lk_form, lk_staging):
    """Identical images: every mismatch is 0, so each level stops after its first iteration.  The intent is a consumer
    level far shorter than the producers' build of the next one, so that the consumers wait at the hand-over; that timing
    is not observable here, only that one iteration per level gives cv2's result bit for bit."""
    a = make_texture_image(11, W, H, contrast=1.2)
    rng = np.random.default_rng(11)
    pts = np.stack([rng.uniform(40, W - 40, 300), rng.uniform(40, H - 40, 300)], 1).astype(np.float32)
    for m in (3, 1):
        q_cv, st_cv = check_lk(gf, a, a.copy(), pts, m, lk_form)
        one, _, _ = cv2.calcOpticalFlowPyrLK(a, a.copy(), pts.reshape(-1, 1, 2), None, winSize=(21, 21), maxLevel=m,
                                             criteria=(cv2.TERM_CRITERIA_COUNT, 1, 0.0))
        assert st_cv.all() and np.array_equal(one.reshape(-1, 2), q_cv)     # one iteration per level gives the result


def test_chain_fallback_on_a_coarse_level(gf, lk_form, lk_staging):
    """A clipped, high-contrast texture under a shift: the first iteration at level 3 exceeds the integer bound of some
    b chain and runs OpenCV's sequential chains (in the two-role form while the producers build level 2)."""
    a = make_texture_image(5, W, H, contrast=5.0)
    b = warp_image(a, 6.0, -5.0, 1.0)
    PI, PJ = pyramid(a), pyramid(b)
    cand = [(x, y) for y in range(120, H - 120, 8) for x in range(120, W - 120, 8)]
    pts = []
    for x, y in cand:
        gx, gy, d = window_terms(PI[3], PJ[3], x >> 3, y >> 3)
        me, det = min_eig(gx, gy)
        if me > 2e-4 and det > 1e-6 and not b_chains_exact(gx, gy, d):
            pts.append((x, y))
    assert len(pts) >= 200, len(pts)
    check_lk(gf, a, b, np.array(pts[::4], np.float32), 3, lk_form)


def test_max_level_0(gf, lk_form, lk_staging):
    """One level: no level overlaps another (in the two-role form the producers build it, the consumers iterate it)."""
    a = make_texture_image(21, W, H, contrast=1.5)
    b = warp_image(a, 2.2, 1.7, 0.5)
    rng = np.random.default_rng(21)
    rand = np.stack([rng.uniform(-5, W + 5, 300), rng.uniform(-5, H + 5, 300)], 1).astype(np.float32)
    check_lk(gf, a, b, np.concatenate([rand, boundary_points(W, H, 0)]), 0, lk_form)


def test_tracker_chain_fallbacks_bit_exact(gf, monkeypatch, lk_form, lk_staging):
    """k_track on the clipped high-contrast stream: both b paths run on every pass (forward levels 3..0, reverse 1..0)
    and the tracks match the oracle."""
    from ground_fusion_b200 import synth
    make_texture = synth.make_texture
    monkeypatch.setattr(synth, "make_texture", lambda seed: make_texture(seed, contrast=300.0))
    totals = np.zeros(2, np.int64)

    def on_frame(k, gpu, ref, got):
        per = lk_debug(gpu)
        assert np.array_equal(per[:, 2] + per[:, 3], per[:, 1]), "frame %d" % k
        totals[:] += per[:, 2:4].sum(0)

    _run_sequence(gf, seed=4, n_frames=10, on_frame=on_frame, form=lk_form)
    assert totals[0] > 0 and totals[1] > 0, totals
