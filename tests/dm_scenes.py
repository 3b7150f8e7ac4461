"""Seeded RGB-D frames and keyframe poses for the dense-map tests: depths across the node's [0.1, 7) m range and poses that put
world points on both sides of both z-band edges (-0.5 and 2 m)."""
import math

import numpy as np


def frame(seed, w, h):
    """rgb (h, w, 3) uint8 with white patches, depth (h, w) uint16 mm: a tilted plane (0.3 .. 7.5 m), steps, holes and clusters."""
    rng = np.random.default_rng(seed)
    ys, xs = np.mgrid[0:h, 0:w]
    d = 300.0 + 7200.0 * (0.6 * xs / w + 0.4 * ys / h)
    d += 400.0 * np.sign(np.sin(xs / 7.0 + seed))
    d = np.rint(d + rng.normal(0, 3, d.shape))
    d[rng.random(d.shape) < 0.05] = 0
    d[rng.random(d.shape) < 0.03] = 50                       # below 0.1 m
    depth = np.clip(d, 0, 65535).astype(np.uint16)
    rgb = rng.integers(0, 256, (h, w, 3)).astype(np.uint8)
    for _ in range(6):
        y, x = int(rng.integers(0, h - 8)), int(rng.integers(0, w - 8))
        rgb[y:y + 8, x:x + 8] = rng.integers(241, 256)
        rgb[y + 8:y + 10, x:x + 8, 2] = 240                  # one channel at the threshold: kept
    return rgb, depth


def rot(rx, ry, rz):
    cx, sx, cy, sy, cz, sz = math.cos(rx), math.sin(rx), math.cos(ry), math.sin(ry), math.cos(rz), math.sin(rz)
    return (np.array([[cz, -sz, 0], [sz, cz, 0], [0, 0, 1]]) @ np.array([[cy, 0, sy], [0, 1, 0], [-sy, 0, cy]])
            @ np.array([[1, 0, 0], [0, cx, -sx], [0, sx, cx]]))


def pose(k):
    """Body pose of keyframe k: camera z roughly along world z, offset down so that world z spans -0.9 .. 6 m."""
    t = 0.1 * k
    return rot(0.05 * math.sin(t), 0.08 * math.sin(0.7 * t), 0.3 * t), np.array([0.4 * math.sin(t), 0.3 * math.cos(0.5 * t), -1.0 + 0.05 * math.sin(t)])


def perturbed(Rs, Ps, seed, scale=0.02):
    """A loop correction: a smooth drift removed along the trajectory."""
    rng = np.random.default_rng(seed)
    n = len(Rs)
    dyaw, dp = rng.normal(0, scale, 1)[0], rng.normal(0, scale, 3)
    out_R = np.array([rot(0, 0, dyaw * k / max(n, 1)) @ Rs[k] for k in range(n)])
    out_P = np.array([Ps[k] + dp * k / max(n, 1) for k in range(n)])
    return out_R, out_P
