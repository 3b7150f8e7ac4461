"""GPU tests of the two ways LK forms its mismatch vector (run with -m gpu on an H100).

Each LK iteration takes b1/b2 either from exact integer sums of the b terms, when every chain is within the 2^24 bound,
or from OpenCV's sequential float chains (fe_lk.cuh, and fe_lk_single.cuh with its own partial layout).  These tracker
sequences run both paths in k_track, in each LK form, which counts per feature the iterations of each path in the
tracker's debug slots [64 + 8*i + 2] and [+ 3], and are bit-exact against oracle/fe_oracle.py.
"""
import numpy as np
import pytest

from test_fe_gpu import _run_sequence, lk_debug, lk_form  # noqa: F401 (fixture)

pytestmark = pytest.mark.gpu
cv2 = pytest.importorskip("cv2")


def _path_counter():
    """(totals, on_frame): on_frame adds each frame's integer-path and chain-path LK iterations of k_track to totals."""
    totals = np.zeros(2, np.int64)

    def on_frame(k, gpu, ref, got):
        per = lk_debug(gpu)
        assert np.array_equal(per[:, 2] + per[:, 3], per[:, 1]), "frame %d: every iteration takes one of the paths" % k
        totals[:] += per[:, 2:4].sum(0)
    return totals, on_frame


def test_c2_sequence_runs_both_paths(gf, lk_form):
    """BASELINE config C2: most iterations take the integer sums, a few fall back to the chains."""
    totals, on_frame = _path_counter()
    _run_sequence(gf, seed=0, n_frames=20, on_frame=on_frame, form=lk_form)
    fast, chain = totals
    assert fast > 0 and chain > 0, (fast, chain)
    assert fast > chain, (fast, chain)


def test_clipped_high_contrast_sequence_runs_both_paths(gf, monkeypatch, lk_form):
    """The scene texture stretched 5x and clipped to 0 and 255: steep gradients push many chains past the bound."""
    from ground_fusion_b200 import synth
    make_texture = synth.make_texture
    monkeypatch.setattr(synth, "make_texture", lambda seed: make_texture(seed, contrast=300.0))
    totals, on_frame = _path_counter()
    _run_sequence(gf, seed=3, n_frames=12, on_frame=on_frame, form=lk_form)
    fast, chain = totals
    assert fast > 0 and chain > 0, (fast, chain)
