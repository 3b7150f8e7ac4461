"""CPU oracle of the YOLO detector and its test data.

- Darknet: darknet's CPU build (oracle/_ref/libdarknet.so, built by oracle/darknet.mk) through oracle/yolo_harness.c: the
  letterboxed input, every layer's output, and the detections after do_nms_obj, for one BGR8 frame.
- extract(): darknet_ros's box extraction and publishing (YoloObjectDetector.cpp detectInThread and the publishing loop),
  restated with its float / double arithmetic.
- write_weights(): a seeded darknet-format .weights file for any cfg, with batch-norm statistics that keep activations O(1) and
  head biases that put a handful of boxes above threshold.
- cfg_at(): a copy of a cfg with another [net] size.
"""
import ctypes
import os

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CFG_DIR = os.path.join(ROOT, "tests", "golden", "yolo_cfg")
ORACLE = os.path.join(ROOT, "oracle", "_ref", "libyolo_oracle.so")
CFGS = ("yolov2-tiny", "yolov2-tiny-voc", "yolov2", "yolov2-voc", "yolov3", "yolov3-voc")
MAX_BOXES = 100


def cfg_path(name):
    return os.path.join(CFG_DIR, name + ".cfg")


def cfg_at(name, out_dir, width=None, height=None, extra=None):
    """The cfg `name` with [net] width / height replaced (and `extra` lines appended to [net]), written under out_dir."""
    lines = open(cfg_path(name)).read().splitlines()
    out, in_net = [], False
    for ln in lines:
        s = ln.replace(" ", "")
        if s.startswith("["):
            if in_net and extra:
                out.extend(extra)
            in_net = s.startswith("[net]")
        elif in_net and width is not None and s.startswith("width="):
            ln = "width=%d" % width
        elif in_net and height is not None and s.startswith("height="):
            ln = "height=%d" % height
        out.append(ln)
    p = os.path.join(out_dir, "%s_%sx%s.cfg" % (name, width, height))
    with open(p, "w") as f:
        f.write("\n".join(out) + "\n")
    return p


def write_weights(cfg, path, seed=0, obj_bias=-3.0, tw_bias=0.0, tie=False, cls_bias=3.0):
    """darknet .weights (header 0.2.0 and an 8-byte seen counter) for the cfg's convolutional layers.
    Hidden layers: weights N(0, 1 / K), rolling mean ~ 0, rolling variance in [0.4, 0.6], scales in [0.9, 1.1]: the gain of about
    sqrt(2) makes up for what leaky takes, so activations stay O(1) through 75 layers.
    The layer before each [region] / [yolo]: small weights, objectness bias obj_bias (a few cells above threshold at -3), w / h
    bias tw_bias, class 0 (+ anchor) bias cls_bias and the others -4.  tie: the head's weights are zero, so objectness and box
    sizes tie across cells and do_nms_obj's order rests on qsort's handling of ties."""
    from ground_fusion_b200.detector import parse_cfg
    _, layers = parse_cfg(cfg)
    rng = np.random.default_rng(seed)
    parts = [np.array([0, 2, 0], np.int32).tobytes(), np.array([0], np.uint64).tobytes()]
    for i, L in enumerate(layers):
        if L["type"] != "convolutional":
            continue
        n, K = L["n"], L["c"] * L["size"] ** 2
        head = i + 1 < len(layers) and layers[i + 1]["type"] in ("region", "yolo")
        if head:
            H = layers[i + 1]
            E = H["classes"] + 5
            w = (rng.standard_normal((n, K)) * (0.5 / np.sqrt(K))).astype(np.float32)
            b = np.zeros(n, np.float32)
            for a in range(H["num"]):
                b[a * E + 2] = b[a * E + 3] = tw_bias
                b[a * E + 4] = obj_bias + 1.5 * (a - H["num"] // 2)   # the anchors spread, so some land a handful above thresh
                b[a * E + 5: a * E + E] = -4.0
                b[a * E + 5 + (a % H["classes"])] = cls_bias
                w[a * E + 4] *= 8.0                    # objectness varies most across cells
            if tie:
                w[:] = 0
        else:
            w = (rng.standard_normal((n, K)) / np.sqrt(K)).astype(np.float32)
            b = (rng.standard_normal(n) * 0.1).astype(np.float32)
        parts.append(b.tobytes())
        if L["batch_normalize"]:
            # a residual branch (the layer before a [shortcut]) gets a small gain, so 23 residual additions stay O(1)
            res = i + 1 < len(layers) and layers[i + 1]["type"] == "shortcut"
            parts.append(rng.uniform(0.9, 1.1, n).astype(np.float32).tobytes() if not res else
                         rng.uniform(0.1, 0.2, n).astype(np.float32).tobytes())
            parts.append((rng.standard_normal(n) * 0.05).astype(np.float32).tobytes())
            parts.append(rng.uniform(0.4, 0.6, n).astype(np.float32).tobytes())
        parts.append(w.tobytes())
    with open(path, "wb") as f:
        f.write(b"".join(parts))
    return path


def conv_params_expected(cfg, path):
    """The per-layer parameters write_weights wrote, read back in the file's order (biases, scales, mean, variance, weights)."""
    from ground_fusion_b200.detector import parse_cfg
    _, layers = parse_cfg(cfg)
    buf = open(path, "rb").read()
    off = 20
    out = {}
    for i, L in enumerate(layers):
        if L["type"] != "convolutional":
            continue
        n, K = L["n"], L["c"] * L["size"] ** 2
        take = lambda m: np.frombuffer(buf, np.float32, m, off)
        d = {"biases": take(n)}
        off += 4 * n
        if L["batch_normalize"]:
            for k in ("scales", "mean", "var"):
                d[k] = take(n)
                off += 4 * n
        d["weights"] = take(n * K)
        off += 4 * n * K
        out[i] = d
    assert off == len(buf)
    return out


def extract(bbox, prob, frame_w, frame_h):
    """darknet_ros's boxes from the detections after NMS: ([(xmin, ymin, xmax, ymax)], [class], [prob]) or empty lists."""
    f32 = np.float32
    roi = []
    for i in range(len(bbox)):
        x, y, w, h = (f32(v) for v in bbox[i])
        xmin = f32(float(x) - float(w) / 2.0)
        xmax = f32(float(x) + float(w) / 2.0)
        ymin = f32(float(y) - float(h) / 2.0)
        ymax = f32(float(y) + float(h) / 2.0)
        xmin = f32(0) if xmin < 0 else xmin
        ymin = f32(0) if ymin < 0 else ymin
        xmax = f32(1) if xmax > 1 else xmax
        ymax = f32(1) if ymax > 1 else ymax
        for j in range(prob.shape[1]):
            if prob[i, j] != 0:
                xc, yc = (xmin + xmax) / f32(2), (ymin + ymax) / f32(2)
                bw, bh = xmax - xmin, ymax - ymin
                if float(bw) > 0.01 and float(bh) > 0.01:
                    roi.append((xc, yc, bw, bh, f32(prob[i, j]), j))
    if len(roi) == 0 or len(roi) > MAX_BOXES:
        return [], [], []
    boxes, cls, probs = [], [], []
    fw, fh = f32(frame_w), f32(frame_h)
    for c in range(prob.shape[1]):
        for (xc, yc, bw, bh, p, j) in roi:
            if j != c:
                continue
            boxes.append((int((xc - bw / f32(2)) * fw), int((yc - bh / f32(2)) * fh), int((xc + bw / f32(2)) * fw),
                          int((yc + bh / f32(2)) * fh)))
            cls.append(c)
            probs.append(p)
    return boxes, cls, probs


def raw_roi_count(bbox, prob):
    """How many boxes the node's extraction collects before its 1..100 check."""
    n = 0
    f32 = np.float32
    for i in range(len(bbox)):
        x, y, w, h = (f32(v) for v in bbox[i])
        xmin = max(f32(float(x) - float(w) / 2.0), f32(0))
        xmax = min(f32(float(x) + float(w) / 2.0), f32(1))
        ymin = max(f32(float(y) - float(h) / 2.0), f32(0))
        ymax = min(f32(float(y) + float(h) / 2.0), f32(1))
        if float(xmax - xmin) > 0.01 and float(ymax - ymin) > 0.01:
            n += int(np.count_nonzero(prob[i]))
    return n


def oracle_available():
    return os.path.exists(ORACLE)


class Darknet:
    """darknet's CPU build on one network (batch 1), driven as darknet_ros drives it."""

    def __init__(self, cfg, weights=None):
        if not oracle_available():
            raise RuntimeError("%s not built: oracle/darknet.mk needs the reference's darknet sources" % ORACLE)
        L = ctypes.CDLL(ORACLE)
        vp, i, f = ctypes.c_void_p, ctypes.c_int, ctypes.c_float
        L.yh_load.restype = vp
        L.yh_load.argtypes = [ctypes.c_char_p, ctypes.c_char_p]
        for name, args in (("yh_n_layers", [vp]), ("yh_net_size", [vp, vp]), ("yh_layer_info", [vp, i, vp, vp]),
                           ("yh_conv_params", [vp, i, vp, vp, vp, vp, vp]), ("yh_letterbox", [vp, vp, i, i, i, vp]),
                           ("yh_predict", [vp, vp]), ("yh_layer_output", [vp, i, vp]), ("yh_detect", [vp, i, i, f, vp, vp, vp, i])):
            getattr(L, name).argtypes = args
            getattr(L, name).restype = i
        L.yh_free.argtypes = [vp]
        L.yh_free.restype = None
        self._L = L
        self._net = L.yh_load(cfg.encode(), weights.encode() if weights else None)
        whc = (ctypes.c_int * 3)()
        L.yh_net_size(self._net, whc)
        self.w, self.h, self.c = whc[0], whc[1], whc[2]
        self.n = L.yh_n_layers(self._net)
        self.layers = [self.layer_info(k) for k in range(self.n)]
        self.classes = self.layers[-1]["classes"]

    def layer_info(self, k):
        name = ctypes.create_string_buffer(32)
        v = (ctypes.c_int * 15)()
        self._L.yh_layer_info(self._net, k, name, v)
        keys = ("w", "h", "c", "out_w", "out_h", "out_c", "outputs", "n", "size", "stride", "pad", "batch_normalize", "activation",
                "classes", "nweights")
        d = dict(zip(keys, list(v)))
        d["type"] = name.value.decode()
        return d

    def conv_params(self, k):
        L = self.layers[k]
        n = L["n"]
        arr = {key: np.zeros(n, np.float32) for key in ("biases", "scales", "mean", "var")}
        arr["weights"] = np.zeros(L["nweights"], np.float32)
        rc = self._L.yh_conv_params(self._net, k, *(arr[key].ctypes.data for key in ("biases", "scales", "mean", "var", "weights")))
        assert rc == 0
        if not L["batch_normalize"]:
            for key in ("scales", "mean", "var"):
                del arr[key]
        return arr

    def letterbox(self, bgr):
        bgr = np.ascontiguousarray(bgr)
        out = np.zeros((3, self.h, self.w), np.float32)
        self._L.yh_letterbox(self._net, bgr.ctypes.data, bgr.strides[0], bgr.shape[1], bgr.shape[0], out.ctypes.data)
        return out

    def forward(self, bgr):
        """Letterbox + network_predict; returns the input image."""
        x = self.letterbox(bgr)
        self._L.yh_predict(self._net, x.ctypes.data)
        return x

    def layer_output(self, k):
        L = self.layers[k]
        out = np.zeros((L["out_c"], L["out_h"], L["out_w"]), np.float32)
        self._L.yh_layer_output(self._net, k, out.ctypes.data)
        return out

    def detections(self, frame_w, frame_h, thresh):
        cap = 1 << 16
        bbox = np.zeros((cap, 4), np.float32)
        obj = np.zeros(cap, np.float32)
        prob = np.zeros((cap, self.classes), np.float32)
        n = self._L.yh_detect(self._net, frame_w, frame_h, ctypes.c_float(thresh), bbox.ctypes.data, obj.ctypes.data,
                              prob.ctypes.data, cap)
        assert n <= cap
        return bbox[:n], obj[:n], prob[:n]

    def detect(self, bgr, thresh):
        """The node's published boxes for one frame: (boxes (m, 4) int64, class ids, probs)."""
        self.forward(bgr)
        bbox, _, prob = self.detections(bgr.shape[1], bgr.shape[0], thresh)
        b, c, p = extract(bbox, prob, bgr.shape[1], bgr.shape[0])
        return np.array(b, np.int64).reshape(-1, 4), np.array(c, np.int32), np.array(p, np.float32)

    def close(self):
        if self._net:
            self._L.yh_free(self._net)
            self._net = None
