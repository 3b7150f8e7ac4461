"""GPU tests of the early exit of the min-distance rounds (nms_cells, fe_select.cuh).

The rounds stop once the corners wanted, accepted in earlier rounds, outrank every cell head still alive.  The output must
stay cv2.goodFeaturesToTrack's bit for bit for any number of corners wanted, and a run that wants few corners must not take
more rounds than one that wants them all.
"""
import numpy as np
import pytest

from conftest import make_texture_image
from test_fe_edges_gpu import check_gftt

pytestmark = pytest.mark.gpu
cv2 = pytest.importorskip("cv2")


@pytest.mark.parametrize("min_dist,n_kept", [(5, 0), (30, 0), (30, 120), (12, 300)])
def test_few_corners_wanted_match_cv2(gf, min_dist, n_kept):
    w, h = 640, 480
    img = make_texture_image(min_dist + n_kept, w, h, contrast=1.4)
    rng = np.random.default_rng(n_kept + 1)
    kept = np.stack([rng.uniform(1, w - 2, n_kept), rng.uniform(1, h - 2, n_kept)], 1).astype(np.float32)
    full = check_gftt(gf, img, 1024 - n_kept, min_dist, kept)          # as many corners as the tracker can hold
    for k in (1, 2, 5, 17, 60):          # (0 is unlimited for cv2; the tracker never asks for 0)
        info = check_gftt(gf, img, k, min_dist, kept)
        assert info["nms_rounds"] <= full["nms_rounds"], (k, info, full)
        assert info["n_candidates"] == full["n_candidates"]
    assert check_gftt(gf, img, 1, min_dist, kept)["nms_rounds"] < full["nms_rounds"]


def test_tracker_sequence_with_one_feature_short(gf):
    """max_cnt 40 at min_dist 30: most frames want one to a few corners, and the sequence stays bit-exact with the oracle."""
    from test_fe_gpu import _run_sequence
    _run_sequence(gf, seed=9, n_frames=20, max_cnt=40, min_dist=30)
