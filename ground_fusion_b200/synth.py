"""Seeded synthetic RGB-D streams (SURVEY.md section 8(d) "synthetic inputs").

Data generation only -- not on the hot path.  A band-limited noise texture (plus a few bright boxes so
that saturated pixels exist) is placed on a plane and rendered through a moving pinhole camera by a
homography; depth is the exact ray/plane intersection in millimetres (u16, 0 beyond 10 m).
cv2 is used for the warp when it is importable, otherwise a numpy bilinear sampler.
Optionally (dynamic=True) a textured rectangle nearer than the plane moves on its own path through the
scene, a stand-in for a person or vehicle; boxes(k) is its bounding box as a detector reports it.
"""
import math

import numpy as np

# config/realsense/idc_cam.yaml of the reference (PINHOLE: fx fy cx cy, radtan k1 k2 p1 p2): the camera of configs C1-C3
IDC_CAM = dict(fx=6.2097277909374247e+02, fy=6.2212293397677581e+02, cx=3.1175896455154810e+02,
               cy=2.4718077836114819e+02, k1=1.4865749308203452e-01, k2=-4.6815685578576460e-01,
               p1=1.6205585303208318e-03, p2=-8.9101576735577930e-03)


def idc_params8():
    """gf_tracker_cfg.pinhole order: fx fy cx cy k1 k2 p1 p2."""
    c = IDC_CAM
    return [c["fx"], c["fy"], c["cx"], c["cy"], c["k1"], c["k2"], c["p1"], c["p2"]]

try:
    import cv2
except Exception:  # pragma: no cover
    cv2 = None


def _gauss_blur_np(a, sigma):
    r = int(3 * sigma + 0.5)
    k = np.exp(-0.5 * (np.arange(-r, r + 1) / sigma) ** 2)
    k /= k.sum()
    a = np.apply_along_axis(lambda v: np.convolve(np.pad(v, r, mode="wrap"), k, mode="valid"), 1, a)
    a = np.apply_along_axis(lambda v: np.convolve(np.pad(v, r, mode="wrap"), k, mode="valid"), 0, a)
    return a


def make_texture(seed, size=(1536, 2048), sigma=2.0, contrast=60.0):
    rng = np.random.default_rng(seed)
    a = rng.standard_normal(size).astype(np.float32)
    if cv2 is not None:
        a = cv2.GaussianBlur(a, (0, 0), sigma)
    else:
        a = _gauss_blur_np(a, sigma).astype(np.float32)
    a = (a - a.mean()) / a.std()
    tex = np.clip(128.0 + contrast * a, 0, 255)
    # a few saturated boxes (exercise the grey>250 rule) and dark boxes (flat regions)
    for _ in range(24):
        y, x = int(rng.integers(0, size[0] - 60)), int(rng.integers(0, size[1] - 60))
        hh, ww = int(rng.integers(12, 48)), int(rng.integers(12, 48))
        tex[y:y + hh, x:x + ww] = 255.0 if rng.random() < 0.6 else 20.0
    return tex.astype(np.uint8)


def _rot(rx, ry, rz):
    cx, sx, cy, sy, cz, sz = math.cos(rx), math.sin(rx), math.cos(ry), math.sin(ry), math.cos(rz), math.sin(rz)
    Rx = np.array([[1, 0, 0], [0, cx, -sx], [0, sx, cx]])
    Ry = np.array([[cy, 0, sy], [0, 1, 0], [-sy, 0, cy]])
    Rz = np.array([[cz, -sz, 0], [sz, cz, 0], [0, 0, 1]])
    return Rz @ Ry @ Rx


class SyntheticStream:
    """frame(k) -> (t, gray u8 HxW, depth u16 HxW).  Deterministic in (seed, k)."""

    def __init__(self, seed=0, width=640, height=480, fps=30.0, K=None, noise_sigma=1.0,
                 plane_dist=4.0, speed=1.0, dynamic=False):
        self.seed, self.w, self.h, self.fps = seed, width, height, fps
        sc = width / 640.0
        self.K = np.array(K if K is not None else
                          [[620.97277909374247 * sc, 0, 311.75896455154810 * sc],
                           [0, 622.12293397677581 * sc, 247.18077836114819 * sc], [0, 0, 1]], float)
        self.tex = make_texture(seed)
        self.noise_sigma = noise_sigma
        self.d0 = plane_dist
        self.speed = speed
        # texture pixel pitch on the plane (metres/pixel) chosen so the texture is ~1 px per image px
        self.pitch = plane_dist / self.K[0, 0]
        # the moving object: a 0.6 m x 0.44 m textured rectangle parallel to the plane, half way to it (off by default, so that
        # the default stream and the fixtures made from it do not change)
        self.dynamic = dynamic
        if dynamic:
            self.obj_tex = make_texture(seed + 7919, size=(220, 300), contrast=70.0)
            self.obj_z, self.obj_half = 0.5 * plane_dist, (0.30, 0.22)
            self.obj_pitch = 2 * self.obj_half[0] / self.obj_tex.shape[1]

    def object_centre(self, k):
        """World centre of the moving rectangle at frame k: it roughly follows the camera's sway, on a faster path of its own."""
        t = k / self.fps * self.speed
        return np.array([0.6 * math.sin(0.7 * t) + 0.3 * math.sin(2.3 * t + 0.5), 0.2 * math.sin(1.7 * t) + 0.05, self.obj_z])

    def boxes(self, k):
        """The moving rectangle's image bounding box as darknet_ros reports it: [(xmin, ymin, xmax, ymax)] int64, the projected
        corners clamped to the image and truncated to integers; empty when it is out of view or the stream has no object."""
        if not self.dynamic:
            return np.zeros((0, 4), np.int64)
        R, C = self.pose(k)
        c, (hx, hy) = self.object_centre(k), self.obj_half
        P = np.array([[c[0] + sx * hx, c[1] + sy * hy, c[2]] for sx in (-1, 1) for sy in (-1, 1)])
        q = self.K @ R @ (P - C).T
        u, v = q[0] / q[2], q[1] / q[2]
        if u.max() < 0 or v.max() < 0 or u.min() > self.w - 1 or v.min() > self.h - 1:
            return np.zeros((0, 4), np.int64)
        lo = [min(max(u.min(), 0.0), self.w - 1), min(max(v.min(), 0.0), self.h - 1)]
        hi = [min(max(u.max(), 0.0), self.w - 1), min(max(v.max(), 0.0), self.h - 1)]
        return np.array([[int(lo[0]), int(lo[1]), int(hi[0]), int(hi[1])]], np.int64)

    def _composite(self, k, R, C, img, depth_m, dc):
        """Paints the moving rectangle over the plane: where a pixel's ray meets it first, gray from its texture, depth from it."""
        dw = R.T @ dc
        s = (self.obj_z - C[2]) / dw[2]
        c, (hx, hy) = self.object_centre(k), self.obj_half
        X, Y = C[0] + s * dw[0] - (c[0] - hx), C[1] + s * dw[1] - (c[1] - hy)
        on = (s > 0) & (X >= 0) & (X < 2 * hx) & (Y >= 0) & (Y < 2 * hy)
        th, tw = self.obj_tex.shape
        u = np.clip(X[on] / self.obj_pitch, 0, tw - 1.001); v = np.clip(Y[on] / self.obj_pitch, 0, th - 1.001)
        u0, v0 = np.floor(u).astype(int), np.floor(v).astype(int)
        fu, fv = u - u0, v - v0
        T = self.obj_tex.astype(np.float32)
        val = ((1 - fu) * (1 - fv) * T[v0, u0] + fu * (1 - fv) * T[v0, u0 + 1] + (1 - fu) * fv * T[v0 + 1, u0] + fu * fv * T[v0 + 1, u0 + 1])
        img.reshape(-1)[on] = val
        depth_m.reshape(-1)[on] = (s * dc[2])[on]

    def pose(self, k):
        """Camera-from-world rotation R and camera centre C (world), smooth figure-eight-like motion."""
        t = k / self.fps * self.speed
        C = np.array([0.9 * math.sin(0.7 * t), 0.25 * math.sin(1.4 * t), 0.35 * math.sin(0.5 * t)])
        R = _rot(0.03 * math.sin(0.9 * t), 0.12 * math.sin(0.7 * t + 0.3), 0.05 * math.sin(0.6 * t))
        return R, C

    def frame(self, k):
        R, C = self.pose(k)
        th, tw = self.tex.shape
        # world plane Z = d0 ; texture coords (U,V) px -> world (X,Y,d0): X=(U-tw/2)*pitch, Y=(V-th/2)*pitch
        A = np.array([[self.pitch, 0, -tw / 2 * self.pitch], [0, self.pitch, -th / 2 * self.pitch], [0, 0, self.d0]])
        # x_img ~ K R (Xw - C) = K R (A [U V 1]^T - C)
        M = self.K @ R @ (A - np.outer(C, [0, 0, 1]))        # texture px -> image px homography
        Minv = np.linalg.inv(M)
        if cv2 is not None:
            img = cv2.warpPerspective(self.tex, M, (self.w, self.h), flags=cv2.INTER_LINEAR,
                                      borderMode=cv2.BORDER_REFLECT_101).astype(np.float32)
        else:  # numpy bilinear
            ys, xs = np.mgrid[0:self.h, 0:self.w]
            p = Minv @ np.stack([xs.ravel(), ys.ravel(), np.ones(xs.size)])
            u, v = p[0] / p[2], p[1] / p[2]
            u = np.clip(u, 0, tw - 1.001); v = np.clip(v, 0, th - 1.001)
            u0, v0 = np.floor(u).astype(int), np.floor(v).astype(int)
            fu, fv = u - u0, v - v0
            T = self.tex.astype(np.float32)
            img = ((1 - fu) * (1 - fv) * T[v0, u0] + fu * (1 - fv) * T[v0, u0 + 1] +
                   (1 - fu) * fv * T[v0 + 1, u0] + fu * fv * T[v0 + 1, u0 + 1]).reshape(self.h, self.w)
        # depth: ray dir (camera) = K^-1 [x y 1]; world dir = R^T dir; hit plane Z=d0: s = (d0 - Cz)/dir_w.z ; depth = s * dir_c.z = s
        ys, xs = np.mgrid[0:self.h, 0:self.w]
        dc = np.linalg.inv(self.K) @ np.stack([xs.ravel(), ys.ravel(), np.ones(xs.size)])
        dw = R.T @ dc
        s = (self.d0 - C[2]) / dw[2]
        depth_m = (s * dc[2]).reshape(self.h, self.w)
        if self.dynamic:
            img = np.ascontiguousarray(img, np.float32)
            self._composite(k, R, C, img, depth_m, dc)
        if self.noise_sigma > 0:
            rng = np.random.default_rng((self.seed + 1) * 1000003 + k)
            img = img + rng.standard_normal(img.shape).astype(np.float32) * self.noise_sigma
        gray = np.clip(np.rint(img), 0, 255).astype(np.uint8)
        depth = np.where((depth_m > 0) & (depth_m < 10.0), np.rint(depth_m * 1000.0), 0).astype(np.uint16)
        return k / self.fps, gray, depth

    def color(self, k):
        """An RGB8 image of frame k for the dense map, derived from frame(k)'s gray image: the saturated boxes of the texture
        (gray >= 246) are white in all three channels, so the mapping node's white test (> 240) has pixels on both sides."""
        gray = self.frame(k)[1].astype(np.int32)
        rgb = np.stack([gray, gray * 7 // 8 + 32, 255 - gray], axis=-1)
        rgb[gray >= 246] = gray[gray >= 246][:, None]
        return rgb.astype(np.uint8)
