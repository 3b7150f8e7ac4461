"""A pure-Python witness of the grid_mapping tool (support_files/grid_mapping: main.cpp:114-120, grid_mapper.cpp, grid_map.cpp):
one point and one ray step at a time with math.log / math.exp, as the tool's double arithmetic on this host.  It pins the C
oracle's libm mode on small inputs."""
import math

import numpy as np


def _div(a, b):
    if b == 0.0:
        return math.copysign(math.inf, a) if a != 0.0 else math.nan
    return a / b


def _log(x):
    return -math.inf if x == 0.0 else math.log(x)


def _exp(x):
    try:
        return math.exp(x)
    except OverflowError:
        return math.inf


def _mv3(M, x):
    return [M[3 * r] * x[0] + M[3 * r + 1] * x[1] + M[3 * r + 2] * x[2] for r in range(3)]


class GridWitness:
    def __init__(self, ric, tic, size_x, size_y, init_x, init_y, cell_size, p_occ=0.6, p_free=0.4, p_prior=0.5):
        self.ric = [float(v) for v in np.asarray(ric, float).reshape(9)]
        self.tic = [float(v) for v in np.asarray(tic, float).reshape(3)]
        self.sx, self.sy, self.ix, self.iy, self.cs = size_x, size_y, init_x, init_y, float(cell_size)
        self.c = [_log(p / (1.0 - p)) for p in (p_free, p_occ, p_prior)]
        self.bel = [[0.5] * size_y for _ in range(size_x)]
        self.kfs = []

    def _cell(self, x, y):
        fx, fy = x / self.cs, y / self.cs
        if not (math.isfinite(fx) and math.isfinite(fy)):
            return None
        cx, cy = math.floor(fx) + self.ix, math.floor(fy) + self.iy
        if cx < 0 or cy < 0 or cx >= self.sx or cy >= self.sy:
            return None
        return cx, cy

    def _update(self, x, y, kind):
        c = self._cell(x, y)
        if c is None:
            return
        b = self.bel[c[0]][c[1]]
        l = _log(_div(b, 1.0 - b))
        l = l + self.c[kind]
        self.bel[c[0]][c[1]] = 1.0 - _div(1.0, 1 + _exp(l))

    def _ray(self, px, py, T0, T1):
        cs = self.cs
        dx, dy = px - T0, py - T1
        z = math.sqrt(dy * dy + dx * dx)
        cosz, sinz = _div(dx, z), _div(dy, z)
        lx, ly = -1.0, -1.0
        r = 0.0
        while r < z + cs:
            wx = (r * cosz if not math.isnan(cosz) else math.nan) + T0
            wy = (r * sinz if not math.isnan(sinz) else math.nan) + T1
            if not (wx == lx and wy == ly):
                kind = 0 if r < (z - 0.5 * cs) else (2 if r > (z + 0.5 * cs) else 1)
                self._update(wx, wy, kind)
                lx, ly = wx, wy
            r += cs

    def _apply(self, R, P, pts):
        for p in pts:
            a = _mv3(self.ric, [float(p[0]), float(p[1]), float(p[2])])
            a = [a[k] + self.tic[k] for k in range(3)]
            b = _mv3(R, a)
            w = [b[k] + P[k] for k in range(3)]
            if w[2] > 0.5 or w[2] < 0.1:
                continue
            self._ray(w[0], w[1], P[0], P[1])

    def addKeyFrame(self, R, P, points):
        R = [float(v) for v in np.asarray(R, float).reshape(9)]
        P = [float(v) for v in np.asarray(P, float).reshape(3)]
        pts = np.asarray(points, np.float32)[:, :3].copy()
        self.kfs.append((R, P, pts))
        self._apply(R, P, pts)

    def updatePath(self, Rs, Ps):
        assert len(Rs) == len(self.kfs)
        self.bel = [[0.5] * self.sy for _ in range(self.sx)]
        for k, (R, P) in enumerate(zip(Rs, Ps)):
            R = [float(v) for v in np.asarray(R, float).reshape(9)]
            P = [float(v) for v in np.asarray(P, float).reshape(3)]
            self.kfs[k] = (R, P, self.kfs[k][2])
            self._apply(R, P, self.kfs[k][2])

    def bel_array(self):
        return np.array(self.bel, np.float64)
