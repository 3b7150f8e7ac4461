"""CPU: the plain-C restatement of cv::CLAHE::apply (tests/clahe_restate.c) is bit-equal to cv2 4.13's createCLAHE(clip, grid).apply
on 8-bit images.  The CUDA kernels (fe_clahe.cuh) follow the restatement; tests/test_clahe_gpu.py compares them with cv2.

Each targeted input is checked to reach its path: tiles that clip, a non-zero residual of the redistribution, padding of the
histogram source (both when one and when both dimensions do not divide by the grid), no clipping at clip 0."""
import numpy as np
import pytest

cv2 = pytest.importorskip("cv2")

from clahe_ref import clahe, cv2_clahe, parity_image as image  # noqa: E402

SIZES = [(640, 480), (641, 480), (640, 481), (1280, 720), (1920, 1080), (377, 377), (424, 400), (752, 480)]
GRIDS = [(1, 1), (3, 11), (7, 5), (8, 8), (16, 16)]
CLIPS = [40.0, 3.0, 1.0, 0.5, 0.0]


def check(img, clip, grid):
    got, st = clahe(img, clip, grid)
    want = cv2_clahe(img, clip, grid)
    assert np.array_equal(got, want), "%d of %d px differ (%s)" % ((got != want).sum(), got.size, st)
    return st


@pytest.mark.parametrize("w,h", SIZES)
@pytest.mark.parametrize("grid", GRIDS)
def test_restatement_equals_cv2_across_geometries(w, h, grid):
    padded_expected = (w % grid[0] != 0) or (h % grid[1] != 0)
    for kind, clip in (("random", 40.0), ("dark", 3.0), ("flat", 1.0)):
        st = check(image(kind, w, h, seed=w + h), clip, grid)
        assert st["padded"] == padded_expected


@pytest.mark.parametrize("clip", CLIPS)
@pytest.mark.parametrize("kind", ["random", "dark", "flat", "near_constant"])
def test_restatement_equals_cv2_across_clip_limits(clip, kind):
    for (w, h), grid in (((640, 480), (8, 8)), ((641, 480), (8, 8)), ((424, 400), (7, 5))):
        st = check(image(kind, w, h, seed=3), clip, grid)
        if clip == 0.0:
            assert st["limit"] == 0 and st["clipped_tiles"] == 0
        else:
            assert st["limit"] >= 1


def test_targeted_paths_are_reached():
    """The inputs above do reach clipping with a residual, padding of one or both dimensions and the limit floor of 1."""
    st = check(image("flat", 640, 480, 1), 3.0, (8, 8))
    assert st["clipped_tiles"] > 0 and st["residual_tiles"] > 0 and not st["padded"]
    st = check(image("flat", 640, 480, 2), 40.0, (8, 8))
    assert st["clipped_tiles"] > 0 and st["residual_tiles"] > 0     # the default clip limit clips flat patches
    st = check(image("flat", 641, 480, 1), 1.0, (8, 8))             # only the width does not divide: both are padded
    assert st["padded"] and st["clipped_tiles"] > 0 and st["residual_tiles"] > 0
    st = check(image("flat", 640, 481, 1), 1.0, (8, 8))             # only the height does not divide
    assert st["padded"] and st["clipped_tiles"] > 0
    st = check(image("random", 641, 481, 4), 40.0, (3, 11))
    assert st["padded"]
    st = check(image("random", 377, 377, 5), 0.5, (16, 16))         # 24x24 tiles: 0.5 * 576 / 256 = 1.125 -> 1
    assert st["limit"] == 1 and st["clipped_tiles"] == 256


def test_padding_of_the_dividing_dimension_matters():
    """A restatement that padded only the non-dividing side would be a different function: check that the image used here
    tells the two apart, so that the equality above really pins the rule."""
    img = image("dark", 641, 480, 7)
    pad_one = cv2.copyMakeBorder(img, 0, 0, 0, 8 - 641 % 8, cv2.BORDER_REFLECT_101)     # 648 x 480: divides, no more padding
    wrong = cv2_clahe(pad_one, 40.0, (8, 8))[:, :641]
    assert (wrong != cv2_clahe(img, 40.0, (8, 8))).mean() > 0.1
    check(img, 40.0, (8, 8))


@pytest.mark.parametrize("grid", [(1, 1), (16, 16), (8, 8)])
@pytest.mark.parametrize("clip", [40.0, 0.0])
def test_constant_image(grid, clip):
    check(image("constant", 640, 480), clip, grid)
    check(image("constant", 641, 481), clip, grid)
