"""The occupancy grid on the GPU (gf_grid_map_*) bit-identical with the sequential C oracle's shared mode after every call: bel,
the map.png pixels and the OccupancyGrid data."""
import numpy as np
import pytest

import dm_scenes
import gm_scenes
from oracle import gm_oracle

pytestmark = pytest.mark.gpu


def _check(g, o):
    assert g.bel().tobytes() == o.bel().tobytes()
    assert g.image().tobytes() == o.image().tobytes()
    assert g.occupancy().tobytes() == o.occupancy().tobytes()


def _pair(cfg=None, **kw):
    from ground_fusion_b200.grid_map import GridMap
    cfg = dict(cfg or {})
    return GridMap(**cfg, **kw), gm_oracle.GridMapOracle(mode="shared", **cfg)


@pytest.mark.parametrize("w,h", [(640, 480), (1280, 720)])
def test_dense_map_sequence_matches_oracle(w, h):
    """200 keyframes of dm_scenes through the dense map, each keyframe's kept points fed to the grid with the same pose, a loop
    correction after keyframe 100.  The band [0.1, 0.5] is populated."""
    from ground_fusion_b200.dense_map import DenseMap
    p8 = [320.0 * w / 640, 318.5 * w / 640, w / 2 - 0.5, h / 2 + 0.5, 0.0, 0.0, 0.0, 0.0]
    ric, tic = dm_scenes.rot(0.01, -0.02, 0.015), np.array([0.03, -0.01, 0.02])
    dm = DenseMap(w, h, p8, 10, 10, ric, tic, max_points=8 << 20, max_keyframes=256)
    g, o = _pair(dict(ric=ric, tic=tic), max_keyframes=256)
    Rs, Ps, applied = [], [], 0
    for k in range(200):
        rgb, depth = dm_scenes.frame(k, w, h)
        R, P = dm_scenes.pose(k)
        dm.addKeyFrame(R, P, rgb, depth)
        pts = dm.keyframePoints(k)
        g.addKeyFrame(R, P, pts); o.addKeyFrame(R, P, pts)
        applied += g.stats()["applied"]
        Rs.append(R); Ps.append(P)
        if k % 10 == 0 or k in (99, 199):
            _check(g, o)
        if k == 99:
            Rn, Pn = dm_scenes.perturbed(np.array(Rs), np.array(Ps), 5)
            g.updatePath(Rn, Pn); o.updatePath(Rn, Pn)
            _check(g, o)
            Rs, Ps = list(Rn), list(Pn)
    assert applied > 0 and (g.bel() != 0.5).sum() > 1000
    assert g.size()[2] == 200
    g.close(); dm.close()


@pytest.mark.parametrize("name", [s[0] for s in gm_scenes.quirk_scenes()])
def test_quirk_scenes(name):
    _, cfg, kfs = next(s for s in gm_scenes.quirk_scenes() if s[0] == name)
    g, o = _pair(cfg)
    for R, P, pts in kfs:
        g.addKeyFrame(R, P, pts); o.addKeyFrame(R, P, pts)
        _check(g, o)
    moved = [(R, P + np.array([0.013, -0.021, 0.0])) for R, P, _ in kfs]
    g.updatePath(*zip(*moved)); o.updatePath(*zip(*moved))
    _check(g, o)
    g.close()


def _vehicle(n_kf, n_pts=3000):
    ric, tic = gm_scenes.camera_to_body()
    return dict(ric=ric, tic=tic), [gm_scenes.body_pose(k) + (gm_scenes.keyframe_points(k, n_pts),) for k in range(n_kf)]


def test_rebuild_equals_fresh_grid_and_chunking_and_intake():
    """A rebuild equals a fresh grid fed the same keyframes; max_records smaller than one keyframe gives the same bits; device
    points with a row stride of 6 equal host points."""
    import torch
    from ground_fusion_b200.grid_map import GridMap
    cfg, kfs = _vehicle(30)
    g, o = _pair(cfg)
    small = GridMap(**cfg, max_records=1000)
    dev = GridMap(**cfg)
    for R, P, pts in kfs:
        g.addKeyFrame(R, P, pts); o.addKeyFrame(R, P, pts)
        small.addKeyFrame(R, P, pts)
        dev.addKeyFrame(R, P, torch.from_numpy(pts).cuda())
        assert g.stats()["records"] > 1000
    _check(g, o); _check(small, o); _check(dev, o)
    st = g.stats()
    assert st["skipped"] >= 0 and st["longest_run"] >= 1
    Rn = [dm_scenes.rot(0, 0, 0.01 * k) @ R for k, (R, _, _) in enumerate(kfs)]
    Pn = [P + np.array([0.002 * k, -0.001 * k, 0.0]) for k, (_, P, _) in enumerate(kfs)]
    for m in (g, o, small, dev):
        m.updatePath(Rn, Pn)
    fresh = GridMap(**cfg)
    for (_, _, pts), R, P in zip(kfs, Rn, Pn):
        fresh.addKeyFrame(R, P, pts[:, :3].copy())
    _check(g, o); _check(small, o); _check(dev, o); _check(fresh, o)
    for m in (g, small, dev, fresh):
        m.close()


def test_small_grid_most_steps_leave():
    cfg, kfs = _vehicle(15, 2000)
    cfg.update(size_x=30, size_y=20, init_x=10, init_y=12, cell_size=0.1)
    g, o = _pair(cfg, max_records=4096)
    for R, P, pts in kfs:
        g.addKeyFrame(R, P, pts); o.addKeyFrame(R, P, pts)
        _check(g, o)
    g.close()


def test_errors_leave_the_grid_unchanged():
    from ground_fusion_b200._lib import GfError
    from ground_fusion_b200.grid_map import GridMap
    for bad in (dict(size_x=0), dict(size_y=-1), dict(size_x=1 << 15, size_y=1 << 15), dict(cell_size=0.0), dict(cell_size=float("nan")),
                dict(p_occ=1.0), dict(p_free=0.0), dict(p_prior=1.5), dict(max_records=0)):
        with pytest.raises(GfError, match="error -1"):
            GridMap(**bad)
    cfg, kfs = _vehicle(3, 500)
    g, o = _pair(cfg, max_keyframes=2, max_points=1200)
    R, P, pts = kfs[0]
    g.addKeyFrame(R, P, pts); o.addKeyFrame(R, P, pts)
    before = (g.bel().tobytes(), g.size())

    def unchanged():
        assert g.bel().tobytes() == before[0] and g.size() == before[1]

    nan_pts = pts.copy(); nan_pts[7, 1] = np.nan
    for args in ((R, P, nan_pts), (R, P + np.array([np.inf, 0, 0]), pts), (np.full((3, 3), np.nan), P, pts)):
        with pytest.raises(GfError, match="error -1"):
            g.addKeyFrame(*args)
        unchanged()
    import torch
    with pytest.raises(GfError, match="error -1"):
        g.addKeyFrame(R, P, torch.from_numpy(nan_pts).cuda())
    unchanged()
    with pytest.raises(GfError, match="error -1"):                 # keyframe count
        g.updatePath([R, R], [P, P])
    unchanged()
    with pytest.raises(GfError, match="error -1"):                 # a non-finite pose in the rebuild
        g.updatePath([R], [P + np.nan])
    unchanged()
    with pytest.raises(GfError, match="error -4"):                 # max_points
        g.addKeyFrame(R, P, np.concatenate([pts, pts]))
    unchanged()
    far = pts.copy(); far[3, :3] = [1e6, 0.0, 1e6]                 # a ray of more than 2^24 steps (pose 0 is the identity)
    with pytest.raises(GfError, match="error -4"):
        g.addKeyFrame(R, P, far)
    unchanged()
    g.addKeyFrame(*kfs[1]); o.addKeyFrame(*kfs[1])
    before = (g.bel().tobytes(), g.size())
    with pytest.raises(GfError, match="error -4"):                 # max_keyframes
        g.addKeyFrame(*kfs[2])
    unchanged()
    _check(g, o)
    g.close()


def test_replay_feeds_the_grid_after_the_dense_map():
    """replay(..., dense_map=, grid_map=) on the GPU pipeline, and the same replay with the oracles in the maps' place."""
    from ground_fusion_b200.dense_map import DenseMap
    from ground_fusion_b200.estimator import BundleAdjuster
    from ground_fusion_b200.feature_manager import FeatureManager
    from ground_fusion_b200.feature_tracker import FeatureTracker
    from ground_fusion_b200.grid_map import GridMap
    from ground_fusion_b200.replay import replay
    from ground_fusion_b200.synth import IDC_CAM, SyntheticStream
    from oracle.dm_oracle import DenseMapOracle
    cam = dict(IDC_CAM, k1=0.0, k2=0.0, p1=0.0, p2=0.0)
    p8 = [cam[k] for k in ("fx", "fy", "cx", "cy", "k1", "k2", "p1", "p2")]

    class Recorder:
        def __init__(self, m):
            self.m, self.calls = m, []

        def addKeyFrame(self, R, P, points):
            self.calls.append((np.array(R), np.array(P), np.array(points)))
            return self.m.addKeyFrame(R, P, points)

    cfg = dict(size_x=400, size_y=400, init_x=200, init_y=200, cell_size=0.05)
    dm, gm = DenseMap(640, 480, p8, 10, 10), Recorder(GridMap(**cfg))
    gtr, gba = FeatureTracker(640, 480, p8, 150, 30, 1, 1), BundleAdjuster(0)
    out = replay(SyntheticStream(seed=0, plane_dist=2.0), gtr, FeatureManager(device=0, depth_threshold=4.0), gba, 40, dense_map=dm, grid_map=gm)
    gtr.close(); gba.close()
    assert out["grid_map"] is gm and len(gm.calls) == out["n_margin_old"] > 0
    o = gm_oracle.GridMapOracle(mode="shared", **cfg)
    for k, (R, P, pts) in enumerate(gm.calls):
        assert pts.tobytes() == dm.keyframePoints(k).tobytes()
        o.addKeyFrame(R, P, pts)
    _check(gm.m, o)
    # the same replay with the oracles in the maps' place: the same keyframes reach the grid oracle
    odm, ogm = DenseMapOracle(640, 480, p8, 10, 10, np.eye(3), np.zeros(3)), gm_oracle.GridMapOracle(mode="shared", **cfg)
    gtr, gba = FeatureTracker(640, 480, p8, 150, 30, 1, 1), BundleAdjuster(0)
    out = replay(SyntheticStream(seed=0, plane_dist=2.0), gtr, FeatureManager(device=0, depth_threshold=4.0), gba, 40, dense_map=odm, grid_map=ogm)
    gtr.close(); gba.close()
    assert out["grid_map"] is ogm and ogm.size()[2] == len(gm.calls)
    _check(gm.m, ogm)
    gm.m.close(); dm.close()
