"""gf_dense_map_group / gf_grid_map_group on the GPU: after every group call each member's dense map (cloud, colours, filter
result, every keyframe's points) and grid (bel, image, occupancy) are byte-equal to a twin single map given the same calls in the
same order; per-member failures leave the member byte-identical; and replay_group feeds the maps as replay() does."""
import numpy as np
import pytest

import dm_scenes

pytestmark = pytest.mark.gpu

W, H = 640, 480
RIC = dm_scenes.rot(0.01, -0.02, 0.015)
TIC = np.array([0.03, -0.01, 0.02])


def _p8(scale=1.0):
    from ground_fusion_b200.synth import IDC_CAM
    cam = dict(IDC_CAM, k1=0.0, k2=0.0, p1=0.0, p2=0.0)
    p = [cam[k] for k in ("fx", "fy", "cx", "cy", "k1", "k2", "p1", "p2")]
    p[0] *= scale; p[1] *= scale
    return p


def _dense(i, w=W, h=H, **kw):
    """member i's map: intrinsics, extrinsics and capacities differ between members, the sampling geometry does not"""
    from ground_fusion_b200.dense_map import DenseMap
    kw.setdefault("max_points", (1 << 20) + 4096 * i)
    kw.setdefault("max_keyframes", 64 + i)
    return DenseMap(w, h, _p8(1.0 + 0.01 * (i % 5)), 10, 10, RIC if i % 2 else np.eye(3), TIC * (i % 3), **kw)


def _grid(i, **kw):
    from ground_fusion_b200.grid_map import GridMap
    kw.setdefault("max_points", 1 << 21)
    kw.setdefault("max_records", 1 << 20)
    # the camera 1.7 m above the body: the stream's plane at 2 m lands in the grid's height band
    return GridMap(RIC if i % 2 else np.eye(3), TIC * (i % 3) + [0, 0, -1.7], size_x=1500 - 100 * (i % 3), size_y=500 + 20 * (i % 2), p_occ=0.6 + 0.05 * (i % 3), **kw)


def _same_dense(a, b):
    assert a.size() == b.size()
    xa, ca = a.cloud()
    xb, cb = b.cloud()
    assert xa.tobytes() == xb.tobytes() and ca.tobytes() == cb.tobytes()
    assert a.filtered()[2].tobytes() == b.filtered()[2].tobytes()
    for k in range(a.size()[2]):
        assert a.keyframePoints(k).tobytes() == b.keyframePoints(k).tobytes()


def _same_grid(a, b, outputs=False):
    assert a.size() == b.size()
    assert a.bel().tobytes() == b.bel().tobytes()
    if outputs:
        assert a.image().tobytes() == b.image().tobytes() and a.occupancy().tobytes() == b.occupancy().tobytes()


class _Frames:
    """seeded keyframes of member i: SyntheticStream(seed=i) frames with the plane at 2 m, body pose from the stream"""

    def __init__(self, K, w=W, h=H):
        from ground_fusion_b200.synth import SyntheticStream
        self.s = [SyntheticStream(seed=i, width=w, height=h, plane_dist=2.0) for i in range(K)]

    def __call__(self, i, k):
        R, C = self.s[i].pose(3 * k)
        return R.T, C, self.s[i].color(3 * k), self.s[i].frame(3 * k)[2]


@pytest.mark.parametrize("K", [1, 3, 16])
def test_group_matches_single_maps(K):
    """Rounds of group calls over changing subsets: the dense group against single twins; the grids fed on the device from the
    dense group, and a second set fed keyframePoints through addKeyFrames, against single twins fed keyframePoints."""
    from ground_fusion_b200.dense_map import DenseMapGroup
    from ground_fusion_b200.grid_map import GridMapGroup
    fr = _Frames(K)
    dm, dt = [_dense(i) for i in range(K)], [_dense(i) for i in range(K)]
    gd, gh, gt = [_grid(i) for i in range(K)], [_grid(i) for i in range(K)], [_grid(i) for i in range(K)]
    dg, ggd, ggh = DenseMapGroup(dm), GridMapGroup(gd), GridMapGroup(gh)
    rng = np.random.default_rng(K)
    kf = [0] * K
    records = 0
    for r in range(5):
        members = list(range(K)) if r == 0 else sorted(rng.choice(K, size=max(1, int(rng.integers(1, K + 1))), replace=False).tolist())
        if r == 1:
            members = members[::-1]                       # any order
        calls = [fr(i, kf[i]) for i in members]
        n, st = dg.addKeyFrames(members, [c[0] for c in calls], [c[1] for c in calls], [c[2] for c in calls], [c[3] for c in calls])
        assert not st.any()
        for j, i in enumerate(members):
            assert dt[i].addKeyFrame(*calls[j]) == n[j]
        assert not ggd.addDenseKeyFrames(dg, members, [c[0] for c in calls], [c[1] for c in calls]).any()
        pts = [dt[i].keyframePoints(kf[i]) for i in members]
        assert not ggh.addKeyFrames(members, [c[0] for c in calls], [c[1] for c in calls], pts).any()
        for j, i in enumerate(members):
            gt[i].addKeyFrame(calls[j][0], calls[j][1], pts[j])
            kf[i] += 1
        for i in range(K):
            _same_dense(dm[i], dt[i])
            _same_grid(gd[i], gt[i], outputs=(r == 4))
            _same_grid(gh[i], gt[i])
            if i in members:
                assert gd[i].stats() == gt[i].stats()
                records += gd[i].stats()["records"]
    assert sum(d.size()[1] for d in dm) > 0 and records > 0
    for x in [ggh, ggd, dg] + dm + dt + gd + gh + gt:
        x.close()


def test_subsets_of_64_members_on_device_frames():
    """A group of 64 at 160 x 120: every member, single members and random subsets, frames as CUDA tensors."""
    import torch
    from ground_fusion_b200.dense_map import DenseMapGroup
    from ground_fusion_b200.grid_map import GridMapGroup
    K, w, h = 64, 160, 120
    dm = [_dense(i, w, h, max_points=1 << 16) for i in range(K)]
    dt = [_dense(i, w, h, max_points=1 << 16) for i in range(K)]
    gd = [_grid(i, max_points=1 << 17) for i in range(K)]
    gt = [_grid(i, max_points=1 << 17) for i in range(K)]
    dg, gg = DenseMapGroup(dm), GridMapGroup(gd)
    rng = np.random.default_rng(7)
    kf = [0] * K
    for members in [list(range(K)), [5], [63], sorted(rng.choice(K, 20, replace=False).tolist()), list(range(K))[::-1]]:
        calls = []
        for i in members:
            rgb, depth = dm_scenes.frame(kf[i] + i, w, h)
            R, P = dm_scenes.pose(kf[i] + 2 * i)
            calls.append((R, P + [0.01 * i, 0, 0], rgb, depth))
        n, st = dg.addKeyFrames(members, [c[0] for c in calls], [c[1] for c in calls], [torch.from_numpy(c[2]).cuda() for c in calls],
                                [torch.from_numpy(c[3].view(np.int16)).cuda() for c in calls])
        assert not st.any()
        assert not gg.addDenseKeyFrames(dg, members, [c[0] for c in calls], [c[1] for c in calls]).any()
        for j, i in enumerate(members):
            assert dt[i].addKeyFrame(*calls[j]) == n[j]
            gt[i].addKeyFrame(calls[j][0], calls[j][1], dt[i].keyframePoints(kf[i]))
            kf[i] += 1
        for i in set(members) | {0, 31}:
            _same_dense(dm[i], dt[i])
            _same_grid(gd[i], gt[i])
    assert sum(d.size()[0] for d in dm) > 0
    for x in [gg, dg] + dm + dt + gd + gt:
        x.close()


def test_failures_are_per_member_and_argument_errors_change_nothing():
    """One call with a member at max_points, one at max_keyframes and one whose keyframe leaves the octree's box: each gets its
    own status and stays byte-identical; the others match their twins.  Then argument errors."""
    from ground_fusion_b200._lib import GfError
    from ground_fusion_b200.dense_map import DenseMap, DenseMapGroup
    from ground_fusion_b200.grid_map import GridMapGroup
    K = 5
    fr = _Frames(K)
    probe = _dense(1)                                     # member 1's capacity: its first keyframe fits, the second does not
    a1, a2 = probe.addKeyFrame(*fr(1, 0)), probe.addKeyFrame(*fr(1, 1))
    probe.close()
    assert a1 > 0 and a2 > 0
    caps = [dict(), dict(max_points=a1 + a2 - 1), dict(max_keyframes=1), dict(), dict()]
    dm, dt = [_dense(i, **caps[i]) for i in range(K)], [_dense(i, **caps[i]) for i in range(K)]
    gm, gt = [_grid(i, max_keyframes=2 if i == 4 else 64) for i in range(K)], [_grid(i, max_keyframes=2 if i == 4 else 64) for i in range(K)]
    dg, gg = DenseMapGroup(dm), GridMapGroup(gm)
    first = [fr(i, 0) for i in range(K)]
    dg.addKeyFrames([1, 2, 3], [first[i][0] for i in (1, 2, 3)], [first[i][1] for i in (1, 2, 3)], [first[i][2] for i in (1, 2, 3)],
                    [first[i][3] for i in (1, 2, 3)])
    for i in (1, 2, 3):
        dt[i].addKeyFrame(*first[i])
    assert dm[1].size()[0] == a1
    before = [(dm[i].cloud()[0].tobytes(), dm[i].filtered()[2].tobytes(), dm[i].size()) for i in range(K)]
    calls = [fr(i, 1) for i in range(K)]
    calls[3] = (np.eye(3), np.array([0.0, -7000.0, 0.0]), calls[3][2], calls[3][3])   # y below the box
    n, st = dg.addKeyFrames(range(K), [c[0] for c in calls], [c[1] for c in calls], [c[2] for c in calls], [c[3] for c in calls])
    assert list(st) == [0, -4, -4, -1, 0], st
    for i in (1, 2, 3):
        assert (dm[i].cloud()[0].tobytes(), dm[i].filtered()[2].tobytes(), dm[i].size()) == before[i] and n[i] == 0
        _same_dense(dm[i], dt[i])
    for i in (0, 4):
        assert dt[i].addKeyFrame(*calls[i]) == n[i]
        _same_dense(dm[i], dt[i])
    # grid: member 4 at max_keyframes after two keyframes, member 2 with a non-finite point, the rest applied
    pts = [dt[i].keyframePoints(dt[i].size()[2] - 1) if dt[i].size()[2] else np.zeros((0, 6), np.float32) for i in range(K)]
    for rnd in range(3):
        p = [x.copy() for x in pts]
        if rnd == 2:
            p[2] = np.concatenate([p[2], np.array([[np.nan, 0, 1, 0, 0, 0]], np.float32)])
        bel = [g.bel().tobytes() for g in gm]
        st = gg.addKeyFrames(range(K), [c[0] for c in calls], [c[1] for c in calls], p)
        want = [0, 0, -1 if rnd == 2 else 0, 0, -4 if rnd == 2 else 0]
        assert list(st) == want, (rnd, st)
        for i in range(K):
            if want[i]:
                assert gm[i].bel().tobytes() == bel[i]
            else:
                gt[i].addKeyFrame(calls[i][0], calls[i][1], p[i])
            _same_grid(gm[i], gt[i])
    # argument errors: nothing changes
    snap = [(d.cloud()[0].tobytes(), d.size()) for d in dm]
    with pytest.raises(ValueError, match="twice"):
        dg.addKeyFrames([0, 0], [calls[0][0]] * 2, [calls[0][1]] * 2, [calls[0][2]] * 2, [calls[0][3]] * 2)
    import ctypes
    from ground_fusion_b200 import _lib
    with pytest.raises(GfError, match="member 1: the member is listed twice"):   # the library's own check
        mb = np.array([0, 0], np.int32)
        R, P = np.zeros((2, 9)), np.zeros((2, 3))
        vp = ctypes.c_void_p * 2
        fp = calls[0][2].ctypes.data, calls[0][3].ctypes.data
        rp, dp = np.full(2, 3 * W, np.uint64), np.full(2, 2 * W, np.uint64)
        _lib.check(_lib.lib().gf_dense_map_group_add_keyframes(dg._h, mb.ctypes.data, 2, R.ctypes.data, P.ctypes.data, vp(fp[0], fp[0]),
                                                               rp.ctypes.data, vp(fp[1], fp[1]), dp.ctypes.data, 0, None, None))
    with pytest.raises(ValueError, match="out of range"):
        dg.addKeyFrames([K], [calls[0][0]], [calls[0][1]], [calls[0][2]], [calls[0][3]])
    assert [(d.cloud()[0].tobytes(), d.size()) for d in dm] == snap
    other = DenseMap(W, H, _p8(), 5, 10)
    with pytest.raises(GfError, match="member 1: width, height, depth_dist or depth_boundary"):
        DenseMapGroup([dm[0], other])
    with pytest.raises(GfError, match="listed twice"):
        DenseMapGroup([dm[0], dm[0]])
    for x in [gg, dg, other] + dm + dt + gm + gt:
        x.close()


def test_direct_calls_between_group_calls():
    """A member rebuilt with update_poses, and one given a single add_keyframe, between two group calls, still match twins."""
    from ground_fusion_b200.dense_map import DenseMapGroup
    from ground_fusion_b200.grid_map import GridMapGroup
    K = 3
    fr = _Frames(K)
    dm, dt = [_dense(i) for i in range(K)], [_dense(i) for i in range(K)]
    gm, gt = [_grid(i) for i in range(K)], [_grid(i) for i in range(K)]
    dg, gg = DenseMapGroup(dm), GridMapGroup(gm)
    poses = [[] for _ in range(K)]

    def group_round(k):
        calls = [fr(i, k) for i in range(K)]
        dg.addKeyFrames(range(K), [c[0] for c in calls], [c[1] for c in calls], [c[2] for c in calls], [c[3] for c in calls])
        gg.addDenseKeyFrames(dg, range(K), [c[0] for c in calls], [c[1] for c in calls])
        for i in range(K):
            dt[i].addKeyFrame(*calls[i])
            gt[i].addKeyFrame(calls[i][0], calls[i][1], dt[i].keyframePoints(dt[i].size()[2] - 1))
            poses[i].append(calls[i][:2])

    group_round(0); group_round(1)
    Rn, Pn = dm_scenes.perturbed(np.array([p[0] for p in poses[0]]), np.array([p[1] for p in poses[0]]), 3)
    for m in (dm[0], dt[0], gm[0], gt[0]):
        m.updatePath(Rn, Pn)
    extra = fr(1, 7)
    dm[1].addKeyFrame(*extra); dt[1].addKeyFrame(*extra)
    gm[1].addKeyFrame(extra[0], extra[1], dm[1].keyframePoints(2)); gt[1].addKeyFrame(extra[0], extra[1], dt[1].keyframePoints(2))
    group_round(2)
    for i in range(K):
        _same_dense(dm[i], dt[i])
        _same_grid(gm[i], gt[i], outputs=True)
    for x in [gg, dg] + dm + dt + gm + gt:
        x.close()


def test_grid_group_chunks_in_order():
    """A grid group whose members sort at most 2^10 records at once matches unchunked single twins (the grid tests' forward
    camera and ground-vehicle poses)."""
    import gm_scenes
    from ground_fusion_b200.grid_map import GridMap, GridMapGroup
    ric, tic = gm_scenes.camera_to_body()
    K = 3
    gm = [GridMap(ric, tic, p_occ=0.6 + 0.05 * i, max_records=1 << 10) for i in range(K)]
    gt = [GridMap(ric, tic, p_occ=0.6 + 0.05 * i, max_records=1 << 22) for i in range(K)]
    gg = GridMapGroup(gm)
    for k in range(3):
        poses = [gm_scenes.body_pose(k + 5 * i) for i in range(K)]
        pts = [gm_scenes.keyframe_points(k + 5 * i) for i in range(K)]
        for i in range(K):
            gt[i].addKeyFrame(poses[i][0], poses[i][1], pts[i])
        assert not gg.addKeyFrames(range(K), [p[0] for p in poses], [p[1] for p in poses], pts).any()
        for i in range(K):
            _same_grid(gm[i], gt[i], outputs=(k == 2))
            assert gm[i].stats()["records"] == gt[i].stats()["records"] > 1 << 10
    for x in [gg] + gm + gt:
        x.close()


# ---- the whole loop ----
N_FRAMES, SEEDS = 60, [0, 1, 2]


def _gpu_parts():
    from ground_fusion_b200.estimator import BundleAdjuster
    from ground_fusion_b200.feature_tracker import FeatureTracker
    from ground_fusion_b200.feature_window import FeatureWindow
    return FeatureTracker(W, H, _p8(), 150, 30, 1, 1), FeatureWindow(depth_threshold=4.0), BundleAdjuster(0)


def _stream(s):
    from ground_fusion_b200.synth import SyntheticStream
    return SyntheticStream(seed=s, plane_dist=2.0)


def _independent(s, **kw):
    from ground_fusion_b200.replay import replay
    tr, fm, ba = _gpu_parts()
    out = replay(_stream(s), tr, fm, ba, N_FRAMES, **kw)
    tr.close(); fm.close(); ba.close()
    return out


def _group(monkeypatch=None, **kw):
    """replay_group over SEEDS; with monkeypatch, the keyframe calls the dense group made, per stream, are recorded"""
    from ground_fusion_b200.dense_map import DenseMapGroup
    from ground_fusion_b200.replay import replay_group
    calls = {s: [] for s in range(len(SEEDS))}
    if monkeypatch is not None:
        orig = DenseMapGroup.addKeyFrames

        def rec(self, members, Rs, Ps, rgbs, depths):
            for j, i in enumerate(members):
                calls[i].append((np.array(Rs[j]), np.array(Ps[j]), rgbs[j].copy(), depths[j].copy()))
            return orig(self, members, Rs, Ps, rgbs, depths)
        monkeypatch.setattr(DenseMapGroup, "addKeyFrames", rec)
    parts = [_gpu_parts() for _ in SEEDS]
    out = replay_group([_stream(s) for s in SEEDS], [p[0] for p in parts], [p[1] for p in parts], [p[2] for p in parts], N_FRAMES, **kw)
    for p in parts:
        for x in p:
            x.close()
    return out, calls


def _close_trajectories(got, refs, label, capsys):
    """The solve's atomics are not ordered: the bar is three times the run-to-run difference of refs (floor 1e-9 m)."""
    d_run = max(np.linalg.norm(a["P_est"] - b["P_est"], axis=1).max() for a, b in zip(refs[0], refs[1]))
    d_grp = max(min(np.linalg.norm(g["P_est"] - r[i]["P_est"], axis=1).max() for r in refs) for i, g in enumerate(got))
    for i, g in enumerate(got):
        assert (g["n_margin_old"], g["n_margin_second_new"], len(g["P_est"])) == (refs[0][i]["n_margin_old"], refs[0][i]["n_margin_second_new"],
                                                                                  len(refs[0][i]["P_est"]))
        assert g["n_removed"] == refs[0][i]["n_removed"] and g["n_predicted"] == refs[0][i]["n_predicted"]
    with capsys.disabled():
        print("\n%s: group vs reference %.3e m, run to run %.3e m" % (label, d_grp, d_run))
    assert d_grp <= max(3 * d_run, 1e-9), (d_grp, d_run)


def test_whole_loop_with_maps(monkeypatch, capsys):
    """replay_group(dense_maps=, grid_maps=) over K = 3 streams: trajectories as today's replay_group; per stream the keyframes
    replay(dense_map=, grid_map=) adds (same count, poses within the trajectory bar); and each stream's maps byte-equal to single
    twins given the keyframes the group added."""
    from ground_fusion_b200.dense_map import DenseMap
    from ground_fusion_b200.grid_map import GridMap
    K = len(SEEDS)
    dms, gms = [DenseMap(W, H, _p8(), 10, 10) for _ in range(K)], [GridMap() for _ in range(K)]
    got, calls = _group(monkeypatch, dense_maps=dms, grid_maps=gms)
    monkeypatch.undo()
    plain = [_group()[0] for _ in range(2)]
    _close_trajectories(got, plain, "replay_group with maps vs without", capsys)

    class Recorder:
        def __init__(self):
            self.m, self.calls = DenseMap(W, H, _p8(), 10, 10), []

        def addKeyFrame(self, R, P, rgb, depth):
            self.calls.append(np.array(P))
            return self.m.addKeyFrame(R, P, rgb, depth)

        def keyframePoints(self, k):
            return self.m.keyframePoints(k)

    for i, s in enumerate(SEEDS):
        assert got[i]["dense_map"] is dms[i] and got[i]["grid_map"] is gms[i]
        r = Recorder()
        ind = _independent(s, dense_map=r, grid_map=GridMap())
        assert len(calls[i]) == len(r.calls) == dms[i].size()[2] > 0
        assert max(np.abs(c[1] - p).max() for c, p in zip(calls[i], r.calls)) <= 1e-8
        twin, gtwin = DenseMap(W, H, _p8(), 10, 10), GridMap()
        for k, (R, P, rgb, depth) in enumerate(calls[i]):
            twin.addKeyFrame(R, P, rgb, depth)
            gtwin.addKeyFrame(R, P, twin.keyframePoints(k))
        _same_dense(dms[i], twin)
        _same_grid(gms[i], gtwin, outputs=True)
        for x in (twin, gtwin, r.m, ind["grid_map"], dms[i], gms[i]):
            x.close()


@pytest.mark.parametrize("feedback", [False, True])
def test_whole_loop_use_mcc(feedback, capsys):
    """replay_group(use_mcc=True) against K independent replay(use_mcc=True) runs, with and without feedback."""
    got = _group(use_mcc=True, feedback=feedback)[0]
    refs = [[_independent(s, use_mcc=True, feedback=feedback) for s in SEEDS] for _ in range(2)]
    _close_trajectories(got, refs, "replay_group use_mcc feedback=%s" % feedback, capsys)
