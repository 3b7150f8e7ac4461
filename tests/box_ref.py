"""trackImagebox's box test, restated for the tests: the reference's literal cv2 call, the closed form the device code implements,
the probe sets both are compared on, and the CPU oracle of trackImagebox.

The reference (feature_tracker.cpp:564-606 mono, :630-673 RGB-D) copies the int64 fields of darknet_ros_msgs/BoundingBox into
`int`, builds the contour {xmin,ymin},{xmin,ymax},{xmax,ymax},{xmax,ymin} of cv::Point2f and leaves a feature out of featureFrame
when pointPolygonTest(contour, cur_pts[i], true) > 0 for any box.  Everything else is trackImage: the oracle below is
oracle.fe_oracle's trackImage followed by that loop, with cv2.pointPolygonTest called as the reference calls it."""
import numpy as np

from oracle.fe_oracle import FeatureTrackerOracle, FeatureTrackerOracleFast


def wrap32(v):
    """int x = (int64_t)v: the low 32 bits as a signed int (GCC, C++20)."""
    return ((int(v) + 2 ** 31) % 2 ** 32) - 2 ** 31


def contour(box):
    x0, y0, x1, y1 = (wrap32(v) for v in box)
    return np.array([[x0, y0], [x0, y1], [x1, y1], [x1, y0]], np.float32)


def cv2_inside(box, pt):
    import cv2
    return cv2.pointPolygonTest(contour(box), (float(pt[0]), float(pt[1])), True) > 0


def closed_form(boxes, pts):
    """[i] = point i lies strictly inside one of the boxes: min(fx0,fx1) < px < max(fx0,fx1) and the same in y, all in float32
    with fx0 = (float)(int)xmin etc. -- what k_select_finalize evaluates."""
    p = np.asarray(pts, np.float32).reshape(-1, 2)
    out = np.zeros(len(p), bool)
    for b in boxes:
        x0, y0, x1, y1 = (np.float32(wrap32(v)) for v in b)
        out |= (min(x0, x1) < p[:, 0]) & (p[:, 0] < max(x0, x1)) & (min(y0, y1) < p[:, 1]) & (p[:, 1] < max(y0, y1))
    return out


def _edge_probes(box):
    """Every vertex, edge midpoint and their float32 neighbours one ulp away in x and in y, plus the centre."""
    x0, y0, x1, y1 = (np.float32(wrap32(v)) for v in box)
    xs = [x0, x1, np.float32((np.float64(x0) + x1) / 2)]
    ys = [y0, y1, np.float32((np.float64(y0) + y1) / 2)]
    out = []
    for x in xs:
        for y in ys:
            for dx in (-np.inf, 0, np.inf):
                for dy in (-np.inf, 0, np.inf):
                    out.append((np.nextafter(x, np.float32(dx)) if dx else x, np.nextafter(y, np.float32(dy)) if dy else y))
    return np.array(out, np.float32)


def probe_sets(seed=0, n_boxes=2000, n_random=6):
    """(box, points) pairs: image-sized boxes, zero-width / zero-height / inverted boxes, corners near +-2^24 (where int -> float
    rounds) and up to +-2^31, and int64 corners outside int32 (which the reference wraps)."""
    rng = np.random.default_rng(seed)
    out = []
    for i in range(n_boxes):
        kind = i % 6
        if kind == 0:
            b = rng.integers(-50, 700, 4)
        elif kind == 1:                                  # degenerate: zero width or zero height
            b = rng.integers(0, 640, 4)
            b[2 + (i // 6) % 2] = b[(i // 6) % 2]
        elif kind == 2:                                  # inverted: xmax < xmin and / or ymax < ymin
            b = rng.integers(0, 640, 4)
            m = (i // 6) % 3                             # 0: x inverted, 1: y inverted, 2: both
            if m != 1:
                b[[0, 2]] = np.sort(b[[0, 2]])[::-1]
            if m != 0:
                b[[1, 3]] = np.sort(b[[1, 3]])[::-1]
        elif kind == 3:                                  # around 2^24, where consecutive ints share a float
            b = rng.integers(2 ** 24 - 40, 2 ** 24 + 40, 4) * rng.choice([-1, 1], 4)
        elif kind == 4:
            b = rng.integers(-2 ** 31, 2 ** 31, 4)
        else:                                            # int64 outside int32: wrapped by `int xmin = box.xmin`
            b = rng.integers(-2 ** 40, 2 ** 40, 4)
        b = np.asarray(b, np.int64)
        x0, y0, x1, y1 = (float(np.float32(wrap32(v))) for v in b)
        lo_x, hi_x, lo_y, hi_y = min(x0, x1), max(x0, x1), min(y0, y1), max(y0, y1)
        mx, my = max(2.0, 0.1 * (hi_x - lo_x)), max(2.0, 0.1 * (hi_y - lo_y))
        rnd = np.stack([rng.uniform(lo_x - mx, hi_x + mx, n_random), rng.uniform(lo_y - my, hi_y + my, n_random)], 1)
        out.append((b, np.concatenate([_edge_probes(b), rnd.astype(np.float32)], 0)))
    return out


class _Imagebox:
    def trackImagebox(self, cur_time, boxes, img, depth=None):
        """FeatureTracker::trackImagebox: trackImage, then featureFrame without the features strictly inside a box."""
        frame = self.trackImage(cur_time, img, depth)
        contours = [contour(b) for b in boxes]
        import cv2
        out = {}
        for i, fid in enumerate(list(self.ids)):
            fid = int(fid)
            if fid not in frame:                         # depth_cam with an empty depth image: featureFrame is empty anyway
                continue
            pt = (float(self.cur_pts[i][0]), float(self.cur_pts[i][1]))
            if any(cv2.pointPolygonTest(c, pt, True) > 0 for c in contours):
                continue
            out[fid] = frame[fid]
        return out


class FeatureTrackerOracleBox(_Imagebox, FeatureTrackerOracle):
    pass


class FeatureTrackerOracleFastBox(_Imagebox, FeatureTrackerOracleFast):
    pass
