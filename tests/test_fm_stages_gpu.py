"""The FeatureManager kernels on the GPU (gf_fm_triangulate, gf_fm_parallax, gf_fm_back_shift_depth,
gf_fm_reprojection_errors, gf_fm_predict_next) through the C ABI, against the high-precision references of tests/fm_ref.py:
ill-conditioned DLT windows, large world coordinates, non-trivial extrinsics, points near the camera plane, every list length,
landmark counts either side of the kernels' blocks, the exact RGB-D depth bounds, stationary windows and argument errors."""
import ctypes

import numpy as np
import pytest

import fm_ref as R
from ground_fusion_b200 import _lib

pytestmark = pytest.mark.gpu

GF_ERR_INVALID_ARG = -1
WORST = {}
_dp = ctypes.POINTER(ctypes.c_double)
_ip = ctypes.POINTER(ctypes.c_int32)


@pytest.fixture(scope="module")
def L():
    from ground_fusion_b200.feature_manager import FeatureManager
    FeatureManager()                                   # declares the gf_fm_* argument types
    yield _lib.lib()
    print("\nworst H100 ratio per bar: " + ", ".join("%s %.3g (%s)" % (k, v[0], v[1]) for k, v in sorted(WORST.items())))


def note(bar, r, name):
    if r > WORST.get(bar, (0.0, ""))[0]:
        WORST[bar] = (r, name)
    return r <= R.K[bar]


def d(a):
    return None if a is None else a.ctypes.data_as(_dp)


def i32(a):
    return None if a is None else a.ctypes.data_as(_ip)


def triangulate(L, sc, idx=None):
    start, nobs, off, pts, dep, est, flag = sc.arrays(idx)
    Ps, Rs = np.ascontiguousarray(sc.Ps), np.ascontiguousarray(sc.Rs.reshape(-1, 9))
    tic, ric = np.ascontiguousarray(sc.tic, np.float64), np.ascontiguousarray(sc.ric.reshape(9), np.float64)
    e, f = est.copy(), flag.copy()
    rc = L.gf_fm_triangulate(0, len(start), i32(start), i32(nobs), i32(off), int(nobs.sum()), d(pts), d(dep), d(e), i32(f), len(Ps),
                             d(Ps), d(Rs), d(tic), d(ric), sc.depth_threshold, R.INIT_DEPTH)
    assert rc == 0, L.gf_last_error()
    return est, flag, e, f


def check_triangulation(sc, refs, est0, flag0, est, flag, name):
    bad = []
    for k, ref in enumerate(refs):
        e, f = est[k], flag[k]
        if ref["kind"] == "skip":
            if est0[k:k + 1].tobytes() != est[k:k + 1].tobytes() or flag0[k] != f:
                bad.append((k, "skipped landmark changed", est0[k], e, flag0[k], f))
            continue
        # whatever the case: a finite depth whose flag agrees with it
        if not (np.isfinite(e) and ((f == 0 and e == R.INIT_DEPTH) or (f in (1, 2) and 0.1 <= e < np.inf))):
            bad.append((k, "inconsistent", e, f))
            continue
        bar = "dlt" if ref["kind"] == "dlt" else "depth_mean"
        if not np.isfinite(ref["scale"]):
            continue
        want_flag = ref["flag"] if ref["kind"] == "dlt" else (1 if ref["flag"] == 1 else 0)
        if R.flag_pinned(ref, R.K[bar]) and f != want_flag:
            bad.append((k, "flag", f, want_flag, e, ref["d"]))
            continue
        if f in (1, 2):
            if f != (2 if ref["kind"] == "dlt" else 1):
                bad.append((k, "path", f, ref["kind"]))
            elif not note(bar, R.ratio(e, ref["d"], ref["scale"]), name):
                bad.append((k, bar, R.ratio(e, ref["d"], ref["scale"]), e, ref["d"]))
    assert not bad, (name, bad[:8])


ALL = {**R.dlt_scenes(), **R.depth_scenes()}


@pytest.mark.parametrize("name", sorted(ALL))
def test_triangulate_matches_the_reference(L, name):
    sc = ALL[name]
    refs = R.triangulate_ref(sc)
    est0, flag0, est, flag = triangulate(L, sc)
    check_triangulation(sc, refs, est0, flag0, est, flag, name)


@pytest.mark.parametrize("n", R.COUNTS)
def test_triangulate_at_counts_around_the_blocks(L, n):
    sc = R.count_scene()
    idx = R.count_index(n)
    refs = R.triangulate_ref(sc)
    est0, flag0, est, flag = triangulate(L, sc, idx)
    check_triangulation(sc, [refs[i] for i in idx], est0, flag0, est, flag, "count n=%d" % n)


@pytest.mark.parametrize("name", sorted(R.stationary_scenes()))
def test_triangulate_in_a_stationary_window_gives_a_finite_depth(L, name):
    """Bit-identical poses: A has a two-dimensional null space, the depth is not determined.  Flag 2 only with 0.1 <= d < inf,
    anything else INIT_DEPTH with flag 0; no NaN or inf reaches estimated_depth (the solve takes 1 / d)."""
    sc = R.stationary_scenes()[name]
    _, _, est, flag = triangulate(L, sc)
    assert np.all(np.isfinite(est))
    assert np.all(((flag == 2) & (est >= 0.1)) | ((flag == 0) & (est == R.INIT_DEPTH))), (est, flag)


@pytest.mark.parametrize("near", [False, True])
@pytest.mark.parametrize("n", R.COUNTS)
def test_parallax_matches_the_reference(L, n, near):
    pi, pj = R.parallax_case(n, n, near)
    ref, s = R.parallax_ref(pi, pj)
    out = ctypes.c_double(-1.0)
    assert L.gf_fm_parallax(0, n, d(pi), d(pj), ctypes.byref(out)) == 0
    r = R.ratio(out.value, ref, s)
    assert note("parallax", r, "n=%d%s" % (n, " near" if near else "")), r


@pytest.mark.parametrize("offset", R.OFFSETS)
@pytest.mark.parametrize("n", [1, 127, 128, 129, 3000])
def test_back_shift_matches_the_reference(L, n, offset):
    uv, dep, mR, mP, nR, nP = R.back_shift_case(n, offset, n)
    z, s = R.back_shift_ref(uv, dep, mR, mP, nR, nP)
    est = dep.copy()
    a = [np.ascontiguousarray(x, np.float64).ravel() for x in (mR, mP, nR, nP)]
    assert L.gf_fm_back_shift_depth(0, n, d(uv), d(est), d(a[0]), d(a[1]), d(a[2]), d(a[3]), R.INIT_DEPTH) == 0
    pinned = np.abs(z) > R.K["back_shift"] * R.EPS * s
    pos = pinned & (z > 0)
    assert np.all(est[pinned & (z <= 0)] == R.INIT_DEPTH)
    if pos.any():
        r = float((np.abs(est - z) / (R.EPS * s))[pos].max())
        assert note("back_shift", r, "n=%d offset %g" % (n, offset)), r
    # near the new camera plane the decision may go either way, the value may not
    loose = ~pinned
    assert np.all((est[loose] == R.INIT_DEPTH) | (np.abs(est[loose] - z[loose]) <= R.K["back_shift"] * R.EPS * s[loose]))


def reprojection(L, sc):
    start, nobs, off, pts, _, est, _ = sc.arrays()
    Ps, Rs = np.ascontiguousarray(sc.Ps), np.ascontiguousarray(sc.Rs.reshape(-1, 9))
    tic, ric = np.ascontiguousarray(sc.tic, np.float64), np.ascontiguousarray(sc.ric.reshape(9), np.float64)
    n = len(start)
    e2, e3, cnt = np.full(n, np.nan), np.full(n, np.nan), np.full(n, -1, np.int32)
    assert L.gf_fm_reprojection_errors(0, n, i32(start), i32(nobs), i32(off), int(nobs.sum()), d(pts), d(est), len(Ps), d(Ps), d(Rs),
                                       d(tic), d(ric), d(e2), d(e3), i32(cnt)) == 0
    return e2, e3, cnt


@pytest.mark.parametrize("near", [False, True])
@pytest.mark.parametrize("offset,ext", [(0.0, False), (0.0, True), (1e3, True), (1e4, True)])
@pytest.mark.parametrize("n", [1, 63, 64, 65, 127, 128, 129, 2000])
def test_reprojection_errors_match_the_reference(L, n, offset, ext, near):
    sc = R.reproj_case(n, offset, ext, n, near)
    e2, e3, cnt = reprojection(L, sc)
    name = "n=%d offset %g%s%s" % (n, offset, " ric" if ext else "", " near" if near else "")
    for k, (w2, w3, wc, s2, s3) in enumerate(R.reproj_ref(sc)):
        assert cnt[k] == wc
        r2, r3 = R.ratio(e2[k], w2, s2), R.ratio(e3[k], w3, s3)
        assert note("reproj2d", r2, name) and note("reproj3d", r3, name), (k, r2, r3)


@pytest.mark.parametrize("frame_count", [1, 5, 10])
@pytest.mark.parametrize("offset,ext", [(0.0, False), (0.0, True), (1e3, True), (1e4, True)])
@pytest.mark.parametrize("n", [1, 64, 65, 1000])
def test_predict_next_matches_the_reference(L, n, offset, ext, frame_count):
    sc, first, uv, dep = R.predict_case(n, offset, ext, n + frame_count)
    ref, s = R.predict_ref(sc, first, uv, dep, frame_count)
    Ps, Rs = np.ascontiguousarray(sc.Ps), np.ascontiguousarray(sc.Rs.reshape(-1, 9))
    tic, ric = np.ascontiguousarray(sc.tic, np.float64), np.ascontiguousarray(sc.ric.reshape(9), np.float64)
    out = np.full((n, 3), np.nan)
    assert L.gf_fm_predict_next(0, n, i32(first), d(uv), d(dep), len(Ps), frame_count, d(Ps), d(Rs), d(tic), d(ric), d(out)) == 0
    r = float((np.abs(out - ref).max(1) / (R.EPS * s)).max())
    assert note("predict", r, "n=%d offset %g%s fc %d" % (n, offset, " ric" if ext else "", frame_count)), r


def test_argument_errors_issue_no_launch(L):
    sc = R.count_scene()
    start, nobs, off, pts, dep, est, flag = sc.arrays(np.arange(8))
    Ps, Rs = np.ascontiguousarray(sc.Ps), np.ascontiguousarray(sc.Rs.reshape(-1, 9))
    tic, ric = np.ascontiguousarray(sc.tic, np.float64), np.ascontiguousarray(sc.ric.reshape(9), np.float64)
    tot = int(nobs.sum())
    n0 = L.gf_kernel_launch_count()

    def tri(start=start, nobs=nobs, off=off, tot=tot, pts=pts, dep=dep, est=est, flag=flag, nf=11, n=8):
        e, f = (None if est is None else est.copy()), (None if flag is None else flag.copy())
        rc = L.gf_fm_triangulate(0, n, i32(start), i32(nobs), i32(off), tot, d(pts), d(dep), d(e), i32(f), nf, d(Ps), d(Rs), d(tic),
                                 d(ric), sc.depth_threshold, R.INIT_DEPTH)
        if rc == GF_ERR_INVALID_ARG:
            assert np.array_equal(e, est) and np.array_equal(f, flag)          # nothing written back
        return rc
    late = start.copy(); late[3] += 1                                         # start_frame + n_obs > n_frames
    assert tri(start=late) == GF_ERR_INVALID_ARG
    assert tri(tot=tot - 1) == GF_ERR_INVALID_ARG                             # obs_offset + n_obs > n_obs_total
    assert tri(nf=12) == GF_ERR_INVALID_ARG                                   # n_frames > GF_BA_MAX_FRAMES
    for k in ("start", "nobs", "off", "pts", "dep", "est", "flag"):
        assert tri(**{k: None}) == GF_ERR_INVALID_ARG, k
    e2, e3, cnt = np.zeros(8), np.zeros(8), np.zeros(8, np.int32)

    def rep(start=start, nobs=nobs, off=off, tot=tot, pts=pts, est=np.full(8, 2.0), e2=e2, e3=e3, cnt=cnt, nf=11):
        return L.gf_fm_reprojection_errors(0, 8, i32(start), i32(nobs), i32(off), tot, d(pts), d(est), nf, d(Ps), d(Rs), d(tic), d(ric),
                                           d(e2), d(e3), i32(cnt))
    assert rep(start=late) == GF_ERR_INVALID_ARG
    assert rep(tot=tot - 1) == GF_ERR_INVALID_ARG
    assert rep(nf=12) == GF_ERR_INVALID_ARG
    for k in ("start", "nobs", "off", "pts", "est", "e2", "e3", "cnt"):
        assert rep(**{k: None}) == GF_ERR_INVALID_ARG, k
    first, uv, dd, out = np.zeros(4, np.int32), np.ones((4, 3)), np.ones(4), np.zeros((4, 3))

    def pred(fc=5, nf=11, first=first, uv=uv, dd=dd, out=out):
        return L.gf_fm_predict_next(0, 4, i32(first), d(uv), d(dd), nf, fc, d(Ps), d(Rs), d(tic), d(ric), d(out))
    for fc in (0, 11, -1):                                                    # frame_count outside [1, n_frames)
        assert pred(fc=fc) == GF_ERR_INVALID_ARG, fc
    assert pred(nf=12) == GF_ERR_INVALID_ARG
    for k in ("first", "uv", "dd", "out"):
        assert pred(**{k: None}) == GF_ERR_INVALID_ARG, k
    s = ctypes.c_double(0)
    assert L.gf_fm_parallax(0, 4, None, d(uv), ctypes.byref(s)) == GF_ERR_INVALID_ARG
    assert L.gf_fm_parallax(0, 4, d(uv), None, ctypes.byref(s)) == GF_ERR_INVALID_ARG
    assert L.gf_fm_parallax(0, 4, d(uv), d(uv), None) == GF_ERR_INVALID_ARG
    R9, P3 = np.eye(3).ravel(), np.zeros(3)
    assert L.gf_fm_back_shift_depth(0, 4, None, d(dd.copy()), d(R9), d(P3), d(R9), d(P3), R.INIT_DEPTH) == GF_ERR_INVALID_ARG
    assert L.gf_fm_back_shift_depth(0, 4, d(uv), None, d(R9), d(P3), d(R9), d(P3), R.INIT_DEPTH) == GF_ERR_INVALID_ARG
    assert L.gf_fm_back_shift_depth(0, 4, d(uv), d(dd.copy()), None, d(P3), d(R9), d(P3), R.INIT_DEPTH) == GF_ERR_INVALID_ARG
    assert L.gf_kernel_launch_count() == n0
