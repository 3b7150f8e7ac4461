import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


def make_texture_image(seed, w=640, h=480, sigma=2.0, contrast=1.0):
    import cv2
    import numpy as np
    rng = np.random.default_rng(seed)
    a = rng.standard_normal((h, w)).astype(np.float32)
    a = cv2.GaussianBlur(a, (0, 0), sigma)
    a = (a - a.mean()) / a.std()
    return np.clip(128 + contrast * 60 * a, 0, 255).astype(np.uint8)


def warp_image(img, dx, dy, ang=0.0):
    import cv2
    h, w = img.shape
    M = cv2.getRotationMatrix2D((w / 2, h / 2), ang, 1.0)
    M[0, 2] += dx
    M[1, 2] += dy
    return cv2.warpAffine(img, M, (w, h), flags=cv2.INTER_LINEAR, borderMode=cv2.BORDER_REFLECT_101)


@pytest.fixture(scope="session")
def gf():
    """The CUDA library through its Python host mirror; fails loudly if it is not built."""
    from ground_fusion_b200 import feature_tracker
    return feature_tracker
