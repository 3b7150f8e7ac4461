"""An independent NumPy / pure-Python restatement of dense_map's colour map for small inputs (tests only): the node's sampling
loop, PoseGraph's z band and voxel-density gate as a sequential dict loop, updatePath's rebuild, and RadiusOutlierRemoval as a
brute-force float32 count of dist^2 < float(0.64)."""
import math

import numpy as np

VOXEL = 0.01


def anchor(lo, hi, res=VOXEL):
    """PCL 1.10 getKeyBitSize on an empty tree (the box widened to 2^depth voxels per axis), from its formula."""
    eps = float(np.finfo(np.float32).eps)
    max_key = max(max(int(math.ceil((h - l - eps) / res)) for l, h in zip(lo, hi)), 2)
    depth = int(math.ceil(math.log2(max_key) - eps))
    side = float(1 << depth) * res
    return [l - (side - (h - l)) / 2.0 for l, h in zip(lo, hi)], [h + (side - (h - l)) / 2.0 for l, h in zip(lo, hi)]


def lift(p8, u, v):
    fx, fy, cx, cy, k1, k2, p1, p2 = p8
    mx_d, my_d = (1.0 / fx) * u + (-cx / fx), (1.0 / fy) * v + (-cy / fy)
    if (k1, k2, p1, p2) == (0.0, 0.0, 0.0, 0.0):
        return mx_d, my_d
    x, y = mx_d, my_d
    for _ in range(8):
        mx2, my2, mxy = x * x, y * y, x * y
        rho2 = mx2 + my2
        rad = k1 * rho2 + k2 * rho2 * rho2
        dx = x * rad + 2.0 * p1 * mxy + p2 * (rho2 + 2.0 * mx2)
        dy = y * rad + 2.0 * p2 * mxy + p1 * (rho2 + 2.0 * my2)
        x, y = mx_d - dx, my_d - dy
    return x, y


def _mv(M, x):
    return [M[i][0] * x[0] + M[i][1] * x[1] + M[i][2] * x[2] for i in range(3)]


def sample(p8, dd, db, rgb, depth):
    """The node's point_rgbd of one frame: list of (x, y, z float32, r, g, b)."""
    h, w = depth.shape
    out = []
    for v in range(db, h - db, dd):
        for u in range(db, w - db, dd):
            d = np.float32(int(depth[v, u])) / np.float32(1000)
            r, g, b = (int(c) for c in rgb[v, u])
            if r > 240 and g > 240 and b > 240:
                continue
            if float(d) < 0.1 or float(d) >= 7.0:
                continue
            ax, ay = lift(p8, float(u), float(v))
            out.append((np.float32(ax * float(d)), np.float32(ay * float(d)), d, r, g, b))
    return out


def world(ric, tic, R, P, l):
    a = _mv(ric, [float(l[0]), float(l[1]), float(l[2])])
    a = [a[i] + tic[i] for i in range(3)]
    b = _mv(R, a)
    return [b[i] + P[i] for i in range(3)]


def key(mn, f):
    return tuple(int((float(f[a]) - mn[a]) / VOXEL) for a in range(3))


class WitnessMap:
    def __init__(self, p8, dd, db, ric, tic):
        self.p8, self.dd, self.db = p8, dd, db
        self.ric, self.tic = [list(map(float, r)) for r in np.asarray(ric)], list(map(float, tic))
        self.mn = anchor((-10000, -1000, -10000), (10000, 10000, 10000))[0]
        self.counts, self.cloud, self.kf = {}, [], []

    def addKeyFrame(self, R, P, rgb, depth):
        R, P = [list(map(float, r)) for r in np.asarray(R)], list(map(float, P))
        kept = []
        for l in sample(self.p8, self.dd, self.db, rgb, depth):
            wv = world(self.ric, self.tic, R, P, l)
            if wv[2] > 2 or wv[2] < -0.5:
                continue
            f = [np.float32(c) for c in wv]
            k = key(self.mn, f)
            if self.counts.get(k, 0) < 3:
                self.counts[k] = self.counts.get(k, 0) + 1
                self.cloud.append((f, l[3:]))
                kept.append(l)
        self.kf.append(kept)
        return len(kept)

    def updatePath(self, Rs, Ps):
        self.mn = anchor((-10000, -10000, -10000), (10000, 10000, 10000))[0]
        self.counts, self.cloud = {}, []
        for pts, R, P in zip(self.kf, Rs, Ps):
            R, P = [list(map(float, r)) for r in np.asarray(R)], list(map(float, P))
            for l in pts:
                f = [np.float32(c) for c in world(self.ric, self.tic, R, P, l)]
                k = key(self.mn, f)
                if self.counts.get(k, 0) < 5:
                    self.counts[k] = self.counts.get(k, 0) + 1
                    self.cloud.append((f, l[3:]))

    def cloud_arrays(self):
        xyz = np.array([c[0] for c in self.cloud], np.float32).reshape(-1, 3)
        rgb = np.array([c[1] for c in self.cloud], np.uint8).reshape(-1, 3)
        return xyz, rgb

    def keyframePoints(self, k):
        return np.array([[float(c) for c in l] for l in self.kf[k]], np.float32).reshape(-1, 6)


def radius_filter(xyz, radius=0.8, min_pts=10):
    """Brute force: keep iff more than min_pts points (itself included) at float32 ((dx*dx) + dy*dy) + dz*dz < float(r^2)."""
    xyz = np.asarray(xyz, np.float32)
    r2 = np.float32(radius * radius)
    keep = np.zeros(len(xyz), bool)
    for i in range(len(xyz)):
        d = xyz[i] - xyz
        d2 = (d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]
        keep[i] = int(np.count_nonzero(d2 < r2)) > min_pts
    return keep
