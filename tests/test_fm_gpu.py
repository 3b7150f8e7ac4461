"""GPU tests of the FeatureManager kernels (csrc/fm_kernels.cu through the C ABI) against oracle/fm_oracle.py, and of the whole
replay pipeline on the GPU (FeatureTracker + FeatureManager + BundleAdjuster) against the same loop driven by the CPU oracles."""
import numpy as np
import pytest

from fm_ref import K, Scene, dlt_ref, ratio
from test_fm_oracle import fill, scene

pytestmark = pytest.mark.gpu


def _gpu_fm(**kw):
    from ground_fusion_b200.feature_manager import FeatureManager
    return FeatureManager(**kw)


@pytest.mark.parametrize("seed,thr,dn", [(1, 0.05, 0.0), (2, 5.0, 0.01), (5, 3.0, 0.02), (6, 10.0, 0.0)])
def test_triangulation_matches_oracle(seed, thr, dn):
    from oracle.fm_oracle import FeatureManagerOracle
    Ps, Rs, lms, frames = scene(seed=seed, n_lm=120, noise=2e-4, depth_noise=dn)
    a, b = FeatureManagerOracle(depth_threshold=thr), _gpu_fm(depth_threshold=thr)
    fill(a, frames); fill(b, frames)
    a.triangulateAll(10, Ps, Rs, np.zeros(3), np.eye(3))
    b.triangulateAll(10, Ps, Rs, np.zeros(3), np.eye(3))
    assert [it.feature_id for it in a.feature] == [it.feature_id for it in b.feature]
    flags = set()
    for x, y in zip(a.feature, b.feature):
        assert x.estimate_flag == y.estimate_flag, x.feature_id
        flags.add(x.estimate_flag)
        if x.estimate_flag == 2:
            # the DLT depth against its high-precision reference and error bar (tests/fm_ref.py)
            lm = dict(start=x.start_frame, pts=np.array([f.point for f in x.feature_per_frame]), dep=np.array([f.depth for f in x.feature_per_frame]))
            want, sc_ = dlt_ref(Scene("", Ps, Rs, np.zeros(3), np.eye(3), thr, [lm]), lm)[:2]
            assert ratio(y.estimated_depth, want, sc_) <= K["dlt"], (x.feature_id, want, y.estimated_depth)
        elif x.estimated_depth > 0:
            assert abs(x.estimated_depth - y.estimated_depth) <= 1e-10 * x.estimated_depth, (x.feature_id, x.estimated_depth, y.estimated_depth)
        else:
            assert y.estimated_depth < 0
    assert len(flags) >= 2
    assert np.allclose(a.getDepthVector(), b.getDepthVector(), rtol=1e-6)
    # window shift with the depth transfer
    a.removeBackShiftDepth(Rs[0], Ps[0], Rs[1], Ps[1]); b.removeBackShiftDepth(Rs[0], Ps[0], Rs[1], Ps[1])
    assert [(it.feature_id, it.start_frame, len(it.feature_per_frame)) for it in a.feature] == [(it.feature_id, it.start_frame, len(it.obs)) for it in b.feature]
    for x, y in zip(a.feature, b.feature):
        if x.estimated_depth > 0:
            assert abs(x.estimated_depth - y.estimated_depth) <= 1e-6 * abs(x.estimated_depth)


def test_keyframe_decision_matches_oracle():
    from oracle.fm_oracle import FeatureManagerOracle
    rng = np.random.default_rng(0)
    a, b = FeatureManagerOracle(), _gpu_fm()
    base = {k: np.array([rng.uniform(-0.4, 0.4), rng.uniform(-0.3, 0.3), 1, 0, 0, 0, 0, 2.0]) for k in range(80)}
    for f in range(11):
        step = 0.004 * f if f < 6 else 0.03 * f                 # slow, then fast image motion
        img = {k: v + np.array([step, 0.3 * step, 0, 0, 0, 0, 0, 0]) for k, v in base.items() if (k + f) % 9}
        ra, rb = a.addFeatureCheckParallax(min(f, 10), img, 0.0), b.addFeatureCheckParallax(min(f, 10), img, 0.0)
        assert ra == rb, f
        assert abs(a.last_average_parallax - b.last_average_parallax) < 1e-9 * max(1.0, a.last_average_parallax)
    assert (a.last_track_num, a.new_feature_num, a.long_track_num) == (b.last_track_num, b.new_feature_num, b.long_track_num)


def test_replay_on_the_gpu_matches_the_oracle_pipeline():
    """The replayed sequence (SURVEY 8(d)): GPU front end + FeatureManager kernels + GPU solver / marginalisations against the CPU
    oracles through the same loop.  The front end is bit-exact and every solve agrees to ~1e-7, so the two trajectories stay
    together far below the 1 mm bar of BASELINE.json; both stay within millimetres of the ground truth."""
    from ground_fusion_b200.estimator import BundleAdjuster
    from ground_fusion_b200.feature_tracker import FeatureTracker
    from ground_fusion_b200.replay import replay
    from ground_fusion_b200.synth import IDC_CAM, SyntheticStream
    from oracle.replay_adapters import oracle_components
    cam = dict(IDC_CAM, k1=0.0, k2=0.0, p1=0.0, p2=0.0)
    p8 = [cam[k] for k in ("fx", "fy", "cx", "cy", "k1", "k2", "p1", "p2")]
    n = 48
    tr, fm, ba = oracle_components(cam, depth_threshold=4.0)
    want = replay(SyntheticStream(seed=0), tr, fm, ba, n)
    gtr, gfm, gba = FeatureTracker(640, 480, p8, 150, 30, 1, 1), _gpu_fm(depth_threshold=4.0), BundleAdjuster(0)
    got = replay(SyntheticStream(seed=0), gtr, gfm, gba, n)
    gtr.close(); gba.close()
    assert (got["n_margin_old"], got["n_margin_second_new"]) == (want["n_margin_old"], want["n_margin_second_new"])
    assert got["iterations"] == want["iterations"]
    d = np.linalg.norm(got["P_est"] - want["P_est"], axis=1)
    assert d.max() < 1e-4, d.max()
    assert abs(got["ate_m"] - want["ate_m"]) < 1e-4 and got["ate_m"] < 5e-3


def test_feedback_loops_match_oracle():
    """gf_fm_reprojection_errors / gf_fm_predict_next behind outliersRejection, movingConsistencyCheckW and predictPtsInNextFrame
    (estimator.cpp:3853-4011) against the oracle's 4x4-transform restatement, with a non-trivial camera extrinsic."""
    from oracle.fm_oracle import FeatureManagerOracle
    Ps, Rs, lms, frames = scene(seed=3, n_lm=150, noise=1e-4)
    a, b = FeatureManagerOracle(depth_threshold=50.0), _gpu_fm(depth_threshold=50.0)
    fill(a, frames); fill(b, frames)
    a.triangulateAll(10, Ps, Rs, np.zeros(3), np.eye(3)); b.triangulateAll(10, Ps, Rs, np.zeros(3), np.eye(3))
    ang = 0.05
    ric = np.array([[np.cos(ang), -np.sin(ang), 0], [np.sin(ang), np.cos(ang), 0], [0, 0, 1.0]])
    tic = np.array([0.02, -0.01, 0.03])
    for k, (x, y) in enumerate(zip(a.feature, b.feature)):       # same depths on both sides, some of them wrong
        y.estimated_depth = x.estimated_depth
        if k % 11 == 5 and x.estimated_depth > 0:
            x.estimated_depth *= 0.4; y.estimated_depth = x.estimated_depth
    wa, wb = a.outliersRejection(Ps, Rs, tic, ric), b.outliersRejection(Ps, Rs, tic, ric)
    assert wa == wb and len(wa) >= 5
    ma, mb = a.movingConsistencyCheckW(Ps, Rs, tic, ric), b.movingConsistencyCheckW(Ps, Rs, tic, ric)
    assert ma == mb and len(ma) >= 5
    feats = [it for it in a.feature if len(it.feature_per_frame) >= 2 and it.estimated_depth > 0]
    gf = [it for it in b.feature if len(it.obs) >= 2 and it.estimated_depth > 0]
    e2, e3, cnt = b._reprojection_errors(gf, Ps, Rs, tic, ric)
    for it, x2, x3, c in zip(feats, e2, e3, cnt):
        w2, w3, wc = a._errors(it, Ps, Rs, tic, ric)
        assert c == wc and abs(x2 - w2) <= 1e-10 * max(1.0, w2) and abs(x3 - w3) <= 1e-10 * max(1.0, w3)
    for fc in (10, 7, 1):
        pa, pb = a.predictPtsInNextFrame(fc, Ps, Rs, tic, ric), b.predictPtsInNextFrame(fc, Ps, Rs, tic, ric)
        assert set(pa) == set(pb) and (fc == 1 or len(pa) > 5)
        for k in pa:
            assert np.allclose(pa[k], pb[k], rtol=1e-11, atol=1e-11), (fc, k)


def test_replay_with_feedback_on_the_gpu():
    """The MULTIPLE_THREAD 0 loop on the GPU components: after every optimisation the GPU tracker gets removeOutliers and the
    prediction computed by gf_fm_predict_next.  The prediction reaches the tracker as float32 pixel positions, so a last-bit
    difference between the two pipelines' FP64 predictions may move an LK start by one ulp: the comparison with the oracle
    pipeline is therefore a millimetre bound, not the 1e-4 m of the feedback-free replay."""
    from ground_fusion_b200.estimator import BundleAdjuster
    from ground_fusion_b200.feature_tracker import FeatureTracker
    from ground_fusion_b200.replay import replay
    from ground_fusion_b200.synth import IDC_CAM, SyntheticStream
    from oracle.replay_adapters import oracle_components
    cam = dict(IDC_CAM, k1=0.0, k2=0.0, p1=0.0, p2=0.0)
    p8 = [cam[k] for k in ("fx", "fy", "cx", "cy", "k1", "k2", "p1", "p2")]
    n = 36
    tr, fm, ba = oracle_components(cam, depth_threshold=4.0)
    want = replay(SyntheticStream(seed=0), tr, fm, ba, n, feedback=True, use_mcc=True)
    gtr, gfm, gba = FeatureTracker(640, 480, p8, 150, 30, 1, 1), _gpu_fm(depth_threshold=4.0), BundleAdjuster(0)
    got = replay(SyntheticStream(seed=0), gtr, gfm, gba, n, feedback=True, use_mcc=True)
    gtr.close(); gba.close()
    assert got["n_predicted"] > 26 * 50 and abs(got["n_predicted"] - want["n_predicted"]) <= 0.02 * want["n_predicted"]
    assert got["ate_m"] < 5e-3 and abs(got["ate_m"] - want["ate_m"]) < 1e-3
    assert np.linalg.norm(got["P_est"] - want["P_est"], axis=1).max() < 2e-3
