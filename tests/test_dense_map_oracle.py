"""The dense map's C oracle (oracle/dm_oracle.c) against an independent NumPy witness on small inputs (no GPU)."""
import numpy as np
import pytest

import dm_scenes
import dm_witness
from oracle import dm_oracle

P8_DIST = [320.0, 318.5, 41.3, 29.7, 0.12, -0.3, 1.5e-3, -8e-3]
P8_PLAIN = [320.0, 318.5, 41.3, 29.7, 0.0, 0.0, 0.0, 0.0]
RIC = dm_scenes.rot(0.01, -0.02, 0.015)
TIC = np.array([0.03, -0.01, 0.02])


def test_octree_anchors_match_pcl_formula():
    for rebuild, lo in ((False, (-10000, -1000, -10000)), (True, (-10000, -10000, -10000))):
        mn, mx = dm_oracle.anchor(rebuild)
        wmn, wmx = dm_witness.anchor(lo, (10000, 10000, 10000))
        assert list(mn) == wmn and list(mx) == wmx
    mn, _ = dm_oracle.anchor(False)
    assert mn[0] == pytest.approx(-10485.76, abs=1e-9) and mn[1] == pytest.approx(-5985.76, abs=1e-9)
    assert dm_oracle.anchor(True)[0][1] == pytest.approx(-10485.76, abs=1e-9)


def _same(o, w, nkf):
    xyz, rgb = o.cloud()
    wxyz, wrgb = w.cloud_arrays()
    assert xyz.tobytes() == wxyz.tobytes() and np.array_equal(rgb, wrgb)
    for k in range(nkf):
        assert o.keyframePoints(k).tobytes() == w.keyframePoints(k).tobytes()
    keep = dm_witness.radius_filter(wxyz)
    assert np.array_equal(o.filtered()[2], np.flatnonzero(keep))


@pytest.mark.parametrize("p8,dd,db", [(P8_DIST, 2, 3), (P8_PLAIN, 3, 0)])
def test_oracle_matches_witness(p8, dd, db):
    w, h = 80, 60
    o = dm_oracle.DenseMapOracle(w, h, p8, dd, db, RIC, TIC)
    wit = dm_witness.WitnessMap(p8, dd, db, RIC, TIC)
    Rs, Ps = [], []
    for k in range(4):
        rgb, depth = dm_scenes.frame(k, w, h)
        R, P = dm_scenes.pose(k)
        # frame 0 three times at one pose (densities saturate at 3), then three times 0.5 m away (fresh voxels)
        for P_ in ([P] * 3 + [P + [0.5, 0, 0]] * 3 if k == 0 else [P]):
            assert o.addKeyFrame(R, P_, rgb, depth) == wit.addKeyFrame(R, P_, rgb, depth)
            Rs.append(R); Ps.append(P_)
        _same(o, wit, len(Rs))
    assert max(wit.counts.values()) == 3
    Rn, Pn = dm_scenes.perturbed(np.array(Rs), np.array(Ps), 1)
    Pn[:, 2] -= 0.3                                       # the correction lowers the map: the rebuild has no z band
    o.updatePath(Rn, Pn)
    wit.updatePath(Rn, Pn)
    _same(o, wit, len(Rs))
    assert o.cloud()[0][:, 2].min() < -0.5
    Ps[3:6] = Ps[:3]                                      # the six copies of frame 0 on one pose: densities saturate at 5
    o.updatePath(Rs, Ps)
    wit.updatePath(Rs, Ps)
    _same(o, wit, len(Rs))
    assert max(wit.counts.values()) == 5


def test_oracle_radius_filter_matches_brute_force():
    rng = np.random.default_rng(3)
    xyz = np.concatenate([rng.normal(0, 0.5, (300, 3)), rng.uniform(-4, 4, (200, 3))]).astype(np.float32)
    xyz = np.concatenate([xyz, xyz[:40]])                 # duplicates count
    assert np.array_equal(dm_oracle.radius_filter(xyz), dm_witness.radius_filter(xyz))


def test_oracle_rejects_points_outside_the_box():
    o = dm_oracle.DenseMapOracle(80, 60, P8_PLAIN, 4, 0, np.eye(3), np.zeros(3))
    rgb, depth = dm_scenes.frame(0, 80, 60)
    with pytest.raises(ValueError):
        o.addKeyFrame(np.eye(3), np.array([0.0, -7000.0, 0.0]), rgb, depth)       # below the constructor's y-min
    assert o.size() == (0, 0, 0)
