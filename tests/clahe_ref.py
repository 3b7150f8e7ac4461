"""CPU references for the front end's `equalize` option -- TEST INFRASTRUCTURE ONLY.

clahe(): ctypes binding of tests/clahe_restate.c, the plain-C restatement of cv::CLAHE::apply (compiled on first use into a
temporary directory, so the source tree is never written).  EqualizingOracle: the reference's trackImage on the image
getImageFromMsg hands it when `equalize` is set, i.e. cv2.createCLAHE(clip, grid).apply(frame) (rosNodeTest.cpp:256-261).
dark_stream(): a dark, low-contrast variant of the synthetic stream, the kind of sequence the option exists for.
"""
import ctypes
import os
import subprocess
import tempfile

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None


def lib():
    global _LIB
    if _LIB is None:
        src = os.path.join(_HERE, "clahe_restate.c")
        so = os.path.join(tempfile.mkdtemp(prefix="gf_clahe_"), "libgf_clahe_restate.so")
        subprocess.check_call(["gcc", "-O2", "-ffp-contract=off", "-msse2", "-mfpmath=sse", "-shared", "-fPIC", "-o", so, src, "-lm"])
        L = ctypes.CDLL(so)
        vp, i = ctypes.c_void_p, ctypes.c_int
        L.gfo_clahe.argtypes = [vp, i, i, ctypes.c_double, i, i, vp, vp]
        L.gfo_clahe.restype = None
        _LIB = L
    return _LIB


def clahe(img, clip=40.0, grid=(8, 8)):
    """Returns (equalised image, stats) with stats = dict(clipped_tiles, residual_tiles, padded, limit)."""
    img = np.ascontiguousarray(img, np.uint8)
    h, w = img.shape
    out = np.empty_like(img)
    st = np.zeros(4, np.int32)
    lib().gfo_clahe(img.ctypes.data, w, h, float(clip), int(grid[0]), int(grid[1]), out.ctypes.data, st.ctypes.data)
    return out, dict(clipped_tiles=int(st[0]), residual_tiles=int(st[1]), padded=bool(st[2]), limit=int(st[3]))


def cv2_clahe(img, clip=40.0, grid=(8, 8)):
    import cv2
    return cv2.createCLAHE(clipLimit=float(clip), tileGridSize=(int(grid[0]), int(grid[1]))).apply(np.ascontiguousarray(img, np.uint8))


def make_equalizing_oracle(clip=40.0, grid=(8, 8)):
    """FeatureTrackerOracle whose trackImage sees the CLAHE'd frame, as the reference's does with `equalize` set: LK on both
    pyramids, goodFeaturesToTrack and the grey > 250 test all read the equalised image."""
    from oracle.fe_oracle import FeatureTrackerOracle

    class EqualizingOracle(FeatureTrackerOracle):
        def trackImage(self, cur_time, img, depth=None):
            return super().trackImage(cur_time, cv2_clahe(img, clip, grid), depth)

    return EqualizingOracle


def darken(gray, gamma=2.2, lo=6, span=48):
    """Gamma plus a contrast squeeze into [lo, lo + span]: a dim, low-contrast frame derived from an ordinary one."""
    g = (gray.astype(np.float64) / 255.0) ** gamma
    return np.clip(np.rint(lo + span * g), 0, 255).astype(np.uint8)


def dark_stream(seed, w, h, n):
    """n frames (t, dark gray, depth) of SyntheticStream(seed) at w x h; the generator itself is left at its defaults."""
    from ground_fusion_b200.synth import SyntheticStream
    st = SyntheticStream(seed=seed, width=w, height=h)
    out = []
    for k in range(n):
        t, g, d = st.frame(k)
        out.append((t, darken(g), d))
    return out


def parity_image(kind, w, h, seed=0):
    """Inputs of the CLAHE parity tests: random, dark (blurred, dim, low contrast), flat (large flat patches: clipping with
    residuals), near_constant, constant."""
    import cv2
    rng = np.random.default_rng(seed)
    if kind == "random":
        return rng.integers(0, 256, (h, w), dtype=np.uint8)
    if kind == "dark":                                   # blurred, dim and low-contrast
        a = cv2.GaussianBlur(rng.standard_normal((h, w)).astype(np.float32), (0, 0), 3.0)
        a = (a - a.mean()) / a.std()
        return darken(np.clip(128 + 60 * a, 0, 255).astype(np.uint8))
    if kind == "flat":                                   # large flat patches on a mild gradient: clipping with residuals
        img = (np.add.outer(np.arange(h) // 7, np.arange(w) // 11) % 40 + 30).astype(np.uint8)
        for _ in range(6):
            y, x = int(rng.integers(0, h - 60)), int(rng.integers(0, w - 80))
            img[y:y + int(rng.integers(30, 200)), x:x + int(rng.integers(40, 300))] = int(rng.integers(0, 256))
        return img
    if kind == "near_constant":
        img = np.full((h, w), 97, np.uint8)
        img[rng.random((h, w)) < 0.002] = 98
        return img
    if kind == "constant":
        return np.full((h, w), 173, np.uint8)
    raise ValueError(kind)
