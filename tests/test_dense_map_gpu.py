"""The dense colour map on the GPU (gf_dense_map_*) bit-identical with the sequential C oracle after every call: the cloud (order,
float bits of xyz, rgb), every keyframe's kept points and the filtered indices."""
import numpy as np
import pytest

import dm_scenes
import dm_witness
from oracle import dm_oracle

pytestmark = pytest.mark.gpu

P8_DIST = [320.0, 318.5, 81.3, 59.7, 0.12, -0.3, 1.5e-3, -8e-3]
P8_PLAIN = [320.0, 318.5, 81.3, 59.7, 0.0, 0.0, 0.0, 0.0]
RIC = dm_scenes.rot(0.01, -0.02, 0.015)
TIC = np.array([0.03, -0.01, 0.02])


def _check(g, o, n_kf, kfs=None, filtered=True, full_recount=True):
    """kfs: the keyframes whose kept points to compare (all when None); filtered: compare the filter's result (the oracle's is
    current)."""
    from ground_fusion_b200.dense_map import radius_filter
    xyz, rgb = g.cloud()
    oxyz, orgb = o.cloud()
    assert xyz.tobytes() == oxyz.tobytes() and np.array_equal(rgb, orgb)
    assert g.size()[0] == o.size()[0] == len(xyz) and g.size()[2] == o.size()[2] == n_kf
    if filtered:
        fx, frgb, idx = g.filtered()
        assert np.array_equal(idx, o.filtered()[2]) and g.size()[1] == len(idx)
        assert fx.tobytes() == xyz[idx].tobytes() and np.array_equal(frgb, rgb[idx])
        if full_recount:                                  # the incremental filter equals a full recount
            assert np.array_equal(np.flatnonzero(radius_filter(xyz)), idx)
    for k in (range(n_kf) if kfs is None else kfs):
        assert g.keyframePoints(k).tobytes() == o.keyframePoints(k).tobytes()


def _pair(w, h, p8, dd, db, ric=RIC, tic=TIC, **kw):
    from ground_fusion_b200.dense_map import DenseMap
    return DenseMap(w, h, p8, dd, db, ric, tic, **kw), dm_oracle.DenseMapOracle(w, h, p8, dd, db, ric, tic)


@pytest.mark.parametrize("w,h", [(640, 480), (1280, 720)])
def test_synthetic_sequence_matches_oracle(w, h):
    """200 keyframes of the synthetic stream with the plane at 2 m (on the z band's upper edge), a loop correction after 100 and
    more keyframes after it.  After every keyframe: the cloud and the new keyframe's list; the filter after every keyframe at
    640x480 (a full recount every 10th) and after every 5th at 1280x720 (the oracle's filter is a full recount of ~1e5-1e6
    points)."""
    from ground_fusion_b200.synth import SyntheticStream, idc_params8
    s = SyntheticStream(seed=0, width=w, height=h, plane_dist=2.0)
    p8 = list(idc_params8())
    p8[0] *= w / 640.0; p8[1] *= w / 640.0; p8[2] *= w / 640.0; p8[3] *= w / 640.0
    g, o = _pair(w, h, p8, 10, 10, np.eye(3), np.zeros(3), max_points=4 << 20, max_keyframes=256)
    every = 1 if w == 640 else 5
    Rs, Ps = [], []
    for k in range(200):
        R, C = s.pose(3 * k)
        rgb, depth = s.color(3 * k), s.frame(3 * k)[2]
        filt = k % every == 0 or k == 199
        assert g.addKeyFrame(R.T, C, rgb, depth) == o.addKeyFrame(R.T, C, rgb, depth, filter=filt)
        Rs.append(R.T); Ps.append(C)
        _check(g, o, k + 1, kfs=[k], filtered=filt, full_recount=(k % 10 == 0))
        if k == 99:
            Rn, Pn = dm_scenes.perturbed(np.array(Rs), np.array(Ps), 5)
            g.updatePath(Rn, Pn); o.updatePath(Rn, Pn)
            _check(g, o, k + 1)
            Rs, Ps = list(Rn), list(Pn)
    _check(g, o, 200)
    assert g.size()[1] > 0
    g.close()


@pytest.mark.parametrize("p8,dd,db,pad,on_device", [(P8_DIST, 1, 0, 0, False), (P8_DIST, 3, 7, 64, False), (P8_PLAIN, 2, 5, 0, True),
                                                     (P8_PLAIN, 5, 1, 32, False), (P8_DIST, 4, 2, 0, True)])
def test_geometry_and_intake_variants(p8, dd, db, pad, on_device):
    import torch
    w, h = 160, 120
    g, o = _pair(w, h, p8, dd, db, max_points=1 << 20, max_keyframes=64)
    Rs, Ps = [], []
    for k in range(12):
        rgb, depth = dm_scenes.frame(k, w, h)
        R, P = dm_scenes.pose(k)
        if on_device:
            grgb, gdepth = torch.from_numpy(rgb).cuda(), torch.from_numpy(depth.view(np.int16)).cuda()
        elif pad:                                         # rows padded beyond the image width
            grgb = np.zeros((h, w + pad, 3), np.uint8)[:, :w]; grgb[...] = rgb
            gdepth = np.zeros((h, w + pad), np.uint16)[:, :w]; gdepth[...] = depth
        else:
            grgb, gdepth = rgb, depth
        assert g.addKeyFrame(R, P, grgb, gdepth) == o.addKeyFrame(R, P, rgb, depth)
        Rs.append(R); Ps.append(P)
        _check(g, o, k + 1)
    Rn, Pn = dm_scenes.perturbed(np.array(Rs), np.array(Ps), 2)
    Pn[:, 2] -= 0.3
    g.updatePath(Rn, Pn); o.updatePath(Rn, Pn)
    _check(g, o, 12)
    assert g.cloud()[0][:, 2].min() < -0.5                # no z band in the rebuild
    g.close()


def test_repeated_frame_saturates_densities():
    """The same frame at one pose, again and again: each voxel takes 3 points; three more copies 0.5 m away fill fresh voxels;
    the rebuild with all six on one pose takes 5 per voxel.  Then loop-corrected poses and further keyframes."""
    w, h = 160, 120
    g, o = _pair(w, h, P8_DIST, 1, 4, max_points=1 << 21, max_keyframes=64)
    rgb, depth = dm_scenes.frame(7, w, h)
    R, P = dm_scenes.pose(3)
    Rs, Ps = [], []
    for i in range(6):
        Pi = P if i < 3 else P + [0.5, 0, 0]
        n = g.addKeyFrame(R, Pi, rgb, depth)
        assert n == o.addKeyFrame(R, Pi, rgb, depth)
        if i in (3, 4, 5):
            assert n > 0
        Rs.append(R); Ps.append(Pi)
        _check(g, o, i + 1)
    assert o.addKeyFrame(R, P, rgb, depth) == g.addKeyFrame(R, P, rgb, depth) == 0     # fourth copy: every voxel holds 3
    Rs.append(R); Ps.append(P)
    _check(g, o, 7)
    Ps = [P] * 7
    g.updatePath(Rs, Ps); o.updatePath(Rs, Ps)
    _check(g, o, 7)
    kp = [len(g.keyframePoints(k)) for k in range(7)]
    assert len(g.cloud()[0]) < sum(kp)                    # the gate < 5 dropped points; the keyframe lists stay as they were
    Rn, Pn = dm_scenes.perturbed(np.array(Rs), np.array(Ps), 9)
    g.updatePath(Rn, Pn); o.updatePath(Rn, Pn)
    _check(g, o, 7)
    for k in range(5):
        rgb2, depth2 = dm_scenes.frame(20 + k, w, h)
        R2, P2 = dm_scenes.pose(20 + k)
        assert g.addKeyFrame(R2, P2, rgb2, depth2) == o.addKeyFrame(R2, P2, rgb2, depth2)
        _check(g, o, 8 + k)
    g.close()


def _boundary_pairs():
    """float32 (dx, dy) whose FLANN distance (dx*dx + dy*dy) + 0*0 equals float(0.8^2) exactly."""
    r2 = np.float32(0.8 * 0.8)
    base = np.float32(0.48)
    dxs = [base]
    for _ in range(64):
        dxs.append(np.nextafter(dxs[-1], np.float32(1)))
    out = []
    for dx in dxs:
        dy = np.float32(np.sqrt(np.float64(r2) - np.float64(dx) * np.float64(dx)))
        for c in (np.nextafter(dy, np.float32(0)), dy, np.nextafter(dy, np.float32(1))):
            if np.float32(dx * dx + c * c) + np.float32(0) == r2:
                out.append((dx, c))
    return out


def test_radius_filter_edges():
    """Points at float squared distance exactly float(0.64) are not neighbours; duplicates and the point itself are."""
    from ground_fusion_b200.dense_map import radius_filter
    pairs = _boundary_pairs()
    assert len(pairs) >= 2
    dx, dy = pairs[0]
    ring = np.array([[sx * a, sy * b, 0] for a, b in ((dx, dy), (dy, dx)) for sx in (1, -1) for sy in (1, -1)], np.float32)
    inside = np.array([[0.1, 0, 0], [0, 0.1, 0]], np.float32)
    for c in ([0, 0, 0], [12.5, -3.0, 0.75], [-0.40625, 0.8125, 1.625]):   # also across filter-cell boundaries
        c = np.array(c, np.float32)
        xyz = np.concatenate([c[None], c + ring, c + inside, c[None]])        # the centre twice: duplicates count
        for min_pts in (3, 4, 11):
            got = radius_filter(xyz, 0.8, min_pts)
            assert np.array_equal(got, dm_oracle.radius_filter(xyz, 0.8, min_pts))
            assert np.array_equal(got, dm_witness.radius_filter(xyz, 0.8, min_pts))
        if not c.any():                                   # centre: itself, its duplicate, 2 inside = 4; the ring is excluded
            assert not radius_filter(xyz, 0.8, 4)[0] and radius_filter(xyz, 0.8, 3)[0]
    rng = np.random.default_rng(0)
    xyz = np.concatenate([rng.normal(0, 0.6, (3000, 3)), rng.uniform(-6, 6, (2000, 3))]).astype(np.float32)
    xyz = np.concatenate([xyz, xyz[:500], np.round(xyz[500:1500] / 0.8125) * 0.8125]).astype(np.float32)
    assert np.array_equal(radius_filter(xyz), dm_oracle.radius_filter(xyz))


def test_points_on_voxel_and_band_boundaries():
    """Keyframe points placed on 1 cm voxel boundaries and on the z band's edges: a flat depth and poses whose offsets are
    multiples of the voxel and land the plane at z = 2 and z = -0.5 exactly (in double)."""
    w, h = 96, 72
    g, o = _pair(w, h, P8_PLAIN, 1, 0, np.eye(3), np.zeros(3), max_points=1 << 20, max_keyframes=32)
    rgb = np.full((h, w, 3), 100, np.uint8)
    n_kf = 0
    for d_mm, Pz in ((2000, 0.0), (2500, -3.0), (1000, -1.5), (1230, 0.77)):
        depth = np.full((h, w), d_mm, np.uint16)
        depth[::3, ::2] = d_mm + 1
        for Px in (0.0, 0.005, 0.01, -0.01):
            P = np.array([Px, -0.02, Pz])
            assert g.addKeyFrame(np.eye(3), P, rgb, depth) == o.addKeyFrame(np.eye(3), P, rgb, depth)
            n_kf += 1
            _check(g, o, n_kf)
    g.close()


def test_errors_leave_the_map_unchanged():
    from ground_fusion_b200._lib import GfError
    from ground_fusion_b200.dense_map import DenseMap
    w, h = 160, 120
    for bad in (dict(depth_dist=0), dict(depth_boundary=60), dict(depth_boundary=80)):
        kw = dict(depth_dist=2, depth_boundary=2)
        kw.update(bad)
        with pytest.raises(GfError, match="error -1"):
            DenseMap(w, h, P8_PLAIN, kw["depth_dist"], kw["depth_boundary"])
    rgb, depth = dm_scenes.frame(1, w, h)
    R, P = dm_scenes.pose(1)

    def unchanged():
        now = (g.cloud(), g.filtered(), g.size(), g.keyframePoints(0))
        assert now[2] == before[2] and now[3].tobytes() == before[3].tobytes()
        assert now[0][0].tobytes() == before[0][0].tobytes() and np.array_equal(now[1][2], before[1][2])

    rgb2, depth2 = dm_scenes.frame(2, w, h)
    R2, P2 = dm_scenes.pose(40)
    g, o = _pair(w, h, P8_DIST, 2, 3, max_points=1 << 20, max_keyframes=2)
    g.addKeyFrame(R, P, rgb, depth); o.addKeyFrame(R, P, rgb, depth)
    before = (g.cloud(), g.filtered(), g.size(), g.keyframePoints(0))
    with pytest.raises(GfError, match="error -1"):        # a point outside the octree's box (y below the constructor's -5985.76)
        g.addKeyFrame(np.eye(3), np.array([0.0, -7000.0, 0.0]), rgb, depth)
    unchanged()
    with pytest.raises(GfError, match="error -1"):        # keyframe count
        g.updatePath([R, R], [P, P])
    unchanged()
    with pytest.raises(GfError, match="error -1"):        # the rebuild's box
        g.updatePath([np.eye(3)], [np.array([0.0, 0.0, -20000.0])])
    unchanged()
    g.addKeyFrame(R2, P2, rgb2, depth2); o.addKeyFrame(R2, P2, rgb2, depth2)
    before = (g.cloud(), g.filtered(), g.size(), g.keyframePoints(0))
    with pytest.raises(GfError, match="error -4"):        # max_keyframes
        g.addKeyFrame(R, P, rgb, depth)
    unchanged()
    _check(g, o, 2)
    g.close()


def test_capacity_error_before_any_change():
    from ground_fusion_b200._lib import GfError
    w, h = 160, 120
    g, o = _pair(w, h, P8_DIST, 2, 3, max_points=4000, max_keyframes=16)
    k = 0
    with pytest.raises(GfError, match="error -4"):
        while True:
            rgb, depth = dm_scenes.frame(k, w, h)
            R, P = dm_scenes.pose(k)
            n_before = g.size()
            g.addKeyFrame(R, P + [0.7 * k, 0, 0], rgb, depth)
            o.addKeyFrame(R, P + [0.7 * k, 0, 0], rgb, depth)
            k += 1
    assert g.size() == n_before
    _check(g, o, k)
    g.close()


def test_replay_feeds_the_map_like_pubkeyframe():
    """replay(..., dense_map=) on the GPU pipeline; the oracle map fed the same keyframe poses and images agrees bit for bit."""
    from ground_fusion_b200.dense_map import DenseMap
    from ground_fusion_b200.estimator import BundleAdjuster
    from ground_fusion_b200.feature_manager import FeatureManager
    from ground_fusion_b200.feature_tracker import FeatureTracker
    from ground_fusion_b200.replay import replay
    from ground_fusion_b200.synth import IDC_CAM, SyntheticStream
    cam = dict(IDC_CAM, k1=0.0, k2=0.0, p1=0.0, p2=0.0)
    p8 = [cam[k] for k in ("fx", "fy", "cx", "cy", "k1", "k2", "p1", "p2")]

    class Recorder:
        def __init__(self, m):
            self.m, self.calls = m, []

        def addKeyFrame(self, R, P, rgb, depth):
            self.calls.append((np.array(R), np.array(P), rgb.copy(), depth.copy()))
            return self.m.addKeyFrame(R, P, rgb, depth)

    rec = Recorder(DenseMap(640, 480, p8, 10, 10))
    gtr, gba = FeatureTracker(640, 480, p8, 150, 30, 1, 1), BundleAdjuster(0)
    out = replay(SyntheticStream(seed=0, plane_dist=2.0), gtr, FeatureManager(device=0, depth_threshold=4.0), gba, 40, dense_map=rec)
    gtr.close(); gba.close()
    assert out["dense_map"] is rec and len(rec.calls) == out["n_margin_old"] > 0
    o = dm_oracle.DenseMapOracle(640, 480, p8, 10, 10, np.eye(3), np.zeros(3))
    for R, P, rgb, depth in rec.calls:
        o.addKeyFrame(R, P, rgb, depth)
    _check(rec.m, o, len(rec.calls))
    assert rec.m.size()[0] > 0
    rec.m.close()
