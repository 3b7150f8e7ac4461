"""YOLO detector on the GPU: the darknet_ros node the reference's use_yolo front end takes its boxes from
(vins_estimator/src/YoloObjectDetector.cpp), over gf_detector_* (include/gf_b200.h).

    det = YoloDetector("yolov3.cfg", "yolov3.weights", thresh=0.3)
    boxes, class_ids, probs = det.detect(bgr)          # boxes (m, 4) int64 xmin, ymin, xmax, ymax, as darknet_ros publishes them
    tracker.trackImagebox(t, boxes, gray, depth)

Several cameras share one detector: set_max_batch(n) once, then detect_batch(frames) runs the forward pass of up to n frames
in one graph launch, each frame's result bit-equal to detect() on it alone.  detect_batch(frames)'s per-frame boxes go to
TrackerGroup.submit(..., boxes=[b for b, _, _ in results]); detect_batch_csr(frames) gives them as the (boxes, box_start) pair
of the C ABI's gf_tracker_group_submit.

The network is read from the user's darknet cfg and .weights at run time.  precision="exact" (the default) is bit-exact with
darknet's CPU build; precision="tf32" runs the convolutions on the tensor cores with TF32-rounded operands (faster, not bit-exact;
DESIGN.md has the error bound), everything else unchanged.  conv_stage() runs one convolution through the detector's kernels.
parse_cfg() gives the layer shapes darknet derives from a cfg, on the host.  No CPU fallback: without a device every call raises.
"""
import ctypes

import numpy as np

from . import _lib

PRECISIONS = {"exact": 0, "tf32": 1}      # GF_DETECTOR_EXACT, GF_DETECTOR_TF32

_LAYER_TYPES = {"convolutional": "convolutional", "conv": "convolutional", "maxpool": "maxpool", "max": "maxpool",
                "route": "route", "reorg": "reorg", "shortcut": "shortcut", "upsample": "upsample", "region": "region",
                "yolo": "yolo"}


def _sections(path):
    secs = []
    with open(path) as f:
        for line in f:
            s = "".join(ch for ch in line if ch not in " \t\n\r")
            if not s or s[0] in "#;":
                continue
            if s[0] == "[":
                secs.append((s[1:s.index("]")] if "]" in s else s[1:], {}))
                continue
            k, _, v = s.partition("=")
            secs[-1][1][k] = v
    return secs


def parse_cfg(path):
    """The layers of a darknet cfg as darknet's constructors size them: a list of dicts with `type` (darknet's name),
    w, h, c (input), out_w, out_h, out_c and outputs, plus the parameters the weights file depends on (n, size, c and
    batch_normalize of a convolutional layer).  Returns (net, layers) with net = dict(w, h, c).  Only the layer types the
    detector supports are sized; another raises ValueError, as creation refuses it."""
    secs = _sections(path)
    if not secs or secs[0][0] not in ("net", "network"):
        raise ValueError("cfg must start with [net]")
    opt = secs[0][1]
    net = {"w": int(opt.get("width", 0)), "h": int(opt.get("height", 0)), "c": int(opt.get("channels", 0))}
    w, h, c = net["w"], net["h"], net["c"]
    layers = []
    for i, (name, o) in enumerate(secs[1:]):
        t = _LAYER_TYPES.get(name)
        if t is None:
            raise ValueError("unsupported layer type [%s]" % name)
        L = {"type": t, "w": w, "h": h, "c": c}
        gi = lambda k, d: int(o.get(k, d))
        if t == "convolutional":
            size, stride = gi("size", 1), gi("stride", 1)
            pad = size // 2 if gi("pad", 0) else gi("padding", 0)
            n = gi("filters", 1)
            L.update(n=n, size=size, stride=stride, pad=pad, batch_normalize=gi("batch_normalize", 0),
                     out_w=(w + 2 * pad - size) // stride + 1, out_h=(h + 2 * pad - size) // stride + 1, out_c=n)
        elif t == "maxpool":
            stride = gi("stride", 1)
            size = gi("size", stride)
            pad = gi("padding", size - 1)
            L.update(size=size, stride=stride, out_w=(w + pad - size) // stride + 1, out_h=(h + pad - size) // stride + 1, out_c=c)
        elif t == "route":
            idx = [int(v) for v in o["layers"].split(",")]
            idx = [i + k if k < 0 else k for k in idx]
            first = layers[idx[0]]
            L.update(inputs=idx, out_w=first["out_w"], out_h=first["out_h"], out_c=sum(layers[k]["out_c"] for k in idx))
        elif t == "reorg":
            s = gi("stride", 1)
            L.update(stride=s, out_w=w // s, out_h=h // s, out_c=c * s * s)
        elif t == "shortcut":
            k = int(o["from"])
            k = i + k if k < 0 else k
            L.update(index=k, out_w=w, out_h=h, out_c=c)
        elif t == "upsample":
            s = gi("stride", 2)
            L.update(stride=s, out_w=w * s, out_h=h * s, out_c=c)
        elif t == "region":
            L.update(classes=gi("classes", 20), num=gi("num", 1), coords=gi("coords", 4), out_w=w, out_h=h, out_c=c)
        elif t == "yolo":
            mask = o.get("mask")
            num = len(mask.split(",")) if mask else gi("num", 1)
            L.update(classes=gi("classes", 20), num=num, out_w=w, out_h=h, out_c=c)
        L["outputs"] = L["out_w"] * L["out_h"] * L["out_c"]
        layers.append(L)
        w, h, c = L["out_w"], L["out_h"], L["out_c"]
    return net, layers


def _frame(bgr):
    """(pointer, pitch, w, h, on_device, keep-alive) of a BGR8 frame: a numpy (h, w, 3) uint8 array with contiguous rows, or a
    CUDA torch tensor of that shape and layout."""
    if hasattr(bgr, "is_cuda") and bgr.is_cuda:
        if bgr.dtype.itemsize != 1 or bgr.dim() != 3 or bgr.shape[2] != 3 or bgr.stride(2) != 1 or bgr.stride(1) != 3:
            raise ValueError("frame must be (h, w, 3) uint8 with contiguous rows")
        return bgr.data_ptr(), bgr.stride(0), bgr.shape[1], bgr.shape[0], 1, bgr
    a = np.asarray(bgr)
    if a.dtype != np.uint8 or a.ndim != 3 or a.shape[2] != 3:
        raise ValueError("frame must be (h, w, 3) uint8")
    if a.strides[2] != 1 or a.strides[1] != 3:
        a = np.ascontiguousarray(a)
    return a.ctypes.data, a.strides[0], a.shape[1], a.shape[0], 0, a


class YoloDetector:
    """darknet_ros's detector for one network on one GPU.  thresh is the node's detection threshold (its yaml's
    threshold / value); the NMS threshold 0.4 and hier 0.5 are the node's constants.  precision: "exact" (bit-exact with
    darknet's CPU build) or "tf32" (tensor-core convolutions); set_precision() switches a live detector."""

    def __init__(self, cfg, weights, thresh=0.3, device=0, precision="exact"):
        if precision not in PRECISIONS:
            raise ValueError("precision must be one of %s" % sorted(PRECISIONS))
        L = _lib.yolo_lib()
        self._L = L
        self._h = ctypes.c_void_p()
        _lib.check_yolo(L.gf_detector_create(ctypes.byref(self._h), device, str(cfg).encode(), str(weights).encode(), ctypes.c_float(thresh)))
        wh = (ctypes.c_int * 2)()
        nl, nc = ctypes.c_int(), ctypes.c_int()
        _lib.check_yolo(L.gf_detector_info(self._h, wh, ctypes.byref(nl), ctypes.byref(nc)))
        self.net_w, self.net_h, self.n_layers, self.classes = wh[0], wh[1], nl.value, nc.value
        self.thresh = thresh
        self.max_batch = 1
        self._boxes = np.zeros((_lib.GF_MAX_BOXES, 4), np.int64)
        self._cls = np.zeros(_lib.GF_MAX_BOXES, np.int32)
        self._prob = np.zeros(_lib.GF_MAX_BOXES, np.float32)
        self.precision = "exact"
        if precision != "exact":
            try:
                self.set_precision(precision)
            except Exception:
                self.close()
                raise

    def set_precision(self, precision):
        """Switch every later detect to "exact" or "tf32".  The first switch to "tf32" makes a TF32-rounded copy of the weights on
        the device (kept, so switching back and forth is cheap)."""
        if precision not in PRECISIONS:
            raise ValueError("precision must be one of %s" % sorted(PRECISIONS))
        _lib.check_yolo(self._L.gf_detector_set_precision(self._h, PRECISIONS[precision]))
        p = ctypes.c_int()
        _lib.check_yolo(self._L.gf_detector_get_precision(self._h, ctypes.byref(p)))
        self.precision = {v: k for k, v in PRECISIONS.items()}[p.value]

    def detect(self, bgr):
        """boxes (m, 4) int64, class_ids (m,) int32, probs (m,) float32 of one BGR8 frame (m = 0 when the node publishes nothing)."""
        ptr, pitch, w, h, on_dev, _keep = _frame(bgr)
        n = ctypes.c_int()
        _lib.check_yolo(self._L.gf_detector_detect(self._h, ptr, pitch, w, h, on_dev, self._boxes.ctypes.data, self._cls.ctypes.data,
                                              self._prob.ctypes.data, _lib.GF_MAX_BOXES, ctypes.byref(n)))
        m = n.value
        return self._boxes[:m].copy(), self._cls[:m].copy(), self._prob[:m].copy()

    def set_max_batch(self, n):
        """Size the per-image buffers for detect_batch of up to n frames (1 <= n <= 64; a detector starts at 1).  The weights
        are shared: each further image costs only its activations (about 217 MiB of layer outputs for yolov3 at 416 x 416)."""
        _lib.check_yolo(self._L.gf_detector_set_max_batch(self._h, int(n)))
        self.max_batch = int(n)

    def _detect_batch(self, frames):
        if len(frames) == 0:
            raise ValueError("detect_batch needs at least one frame")
        fs = [_frame(f) for f in frames]
        on_dev = {f[4] for f in fs}
        if len(on_dev) != 1:
            raise ValueError("the frames of one batch must be all host arrays or all CUDA tensors")
        n = len(fs)
        ptrs = (ctypes.c_void_p * n)(*[f[0] for f in fs])
        pitch = (ctypes.c_size_t * n)(*[f[1] for f in fs])
        w = (ctypes.c_int * n)(*[f[2] for f in fs])
        h = (ctypes.c_int * n)(*[f[3] for f in fs])
        cap = _lib.GF_MAX_BOXES * n
        boxes, cls, prob = np.zeros((cap, 4), np.int64), np.zeros(cap, np.int32), np.zeros(cap, np.float32)
        start = np.zeros(n + 1, np.int32)
        _lib.check_yolo(self._L.gf_detector_detect_batch(self._h, n, ptrs, pitch, w, h, on_dev.pop(), boxes.ctypes.data,
                                                         cls.ctypes.data, prob.ctypes.data, cap, start.ctypes.data))
        m = start[n]
        return boxes[:m], cls[:m], prob[:m], start

    def detect_batch(self, frames):
        """detect() of each frame in one forward pass: a list of (boxes, class_ids, probs), one per frame.  frames: a list of at
        most max_batch BGR8 frames, all numpy arrays or all CUDA tensors, of any sizes."""
        boxes, cls, prob, start = self._detect_batch(frames)
        return [(boxes[a:b].copy(), cls[a:b].copy(), prob[a:b].copy()) for a, b in zip(start[:-1], start[1:])]

    def detect_batch_csr(self, frames):
        """detect_batch's boxes as (boxes (m, 4) int64, box_start (n + 1,) int32): frame i's are boxes[box_start[i]:box_start[i + 1]],
        the layout of the C ABI's gf_tracker_group_submit (TrackerGroup.submit takes per-frame lists, as detect_batch returns)."""
        boxes, _, _, start = self._detect_batch(frames)
        return boxes, start

    def member_layer_output(self, member, i):
        """Layer i's output for frame `member` of the last detect / detect_batch, as layer_output."""
        shape = self.layer_shape(i)
        out = np.empty(shape, np.float32)
        _lib.check_yolo(self._L.gf_detector_member_layer_output(self._h, member, i, out.ctypes.data, out.size))
        return out

    def layer_shape(self, i):
        whc = (ctypes.c_int * 3)()
        _lib.check_yolo(self._L.gf_detector_layer_shape(self._h, i, whc))
        return whc[2], whc[1], whc[0]

    def layer_output(self, i):
        """Layer i's output of the last detect (frame 0 of the last detect_batch) as (c, h, w) float32; i = -1: the letterboxed
        input."""
        shape = self.layer_shape(i)
        out = np.empty(shape, np.float32)
        _lib.check_yolo(self._L.gf_detector_layer_output(self._h, i, out.ctypes.data, out.size))
        return out

    def input_image(self):
        return self.layer_output(-1)

    def last_device_ms(self):
        ms = ctypes.c_float()
        _lib.check_yolo(self._L.gf_detector_last_device_ms(self._h, ctypes.byref(ms)))
        return ms.value

    def layer_times(self, reps=20):
        """Mean device ms of each layer's kernels, re-run `reps` times on the last frame's data (profiling)."""
        ms = np.zeros(self.n_layers, np.float32)
        _lib.check_yolo(self._L.gf_detector_layer_times(self._h, reps, ms.ctypes.data))
        return ms

    def close(self):
        if self._h:
            self._L.gf_detector_destroy(self._h)
            self._h = ctypes.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def letterbox(bgr, net_w, net_h, device=0):
    """The detector's input image for a BGR8 frame, (3, net_h, net_w) float32: darknet's letterbox_image as the node calls it."""
    ptr, pitch, w, h, on_dev, _keep = _frame(bgr)
    out = np.empty((3, net_h, net_w), np.float32)
    _lib.check_yolo(_lib.yolo_lib().gf_stage_letterbox(device, ptr, pitch, w, h, on_dev, net_w, net_h, out.ctypes.data))
    return out


def conv_stage(x, w, bias, stride=1, pad=0, leaky=False, bn=None, precision="exact", device=0):
    """One convolutional layer through the detector's kernels and tile choice for its shape: x (C, H, W), w (M, C, size, size) or
    (M, C size size) with size given by a 4-d w, bias (M,), bn = (scale, mean, var) or None.  Returns (M, OH, OW) float32."""
    if precision not in PRECISIONS:
        raise ValueError("precision must be one of %s" % sorted(PRECISIONS))
    x = np.ascontiguousarray(x, np.float32)
    w = np.asarray(w, np.float32)
    C, H, W = x.shape
    M = w.shape[0]
    size = w.shape[2] if w.ndim == 4 else int(round((w.size // (M * C)) ** 0.5))
    if w.size != M * C * size * size:
        raise ValueError("w must hold M x C x size x size values")
    w = np.ascontiguousarray(w.reshape(M, C * size * size))
    bias = np.ascontiguousarray(bias, np.float32)
    vec = [np.ascontiguousarray(v, np.float32) for v in bn] if bn is not None else []
    if bias.shape != (M,) or any(v.shape != (M,) for v in vec):
        raise ValueError("bias and batch-norm vectors must have M entries")
    OW, OH = (W + 2 * pad - size) // stride + 1, (H + 2 * pad - size) // stride + 1
    out = np.empty((M, OH, OW), np.float32)
    shape = (ctypes.c_int * 9)(C, H, W, M, size, stride, pad, 1 if bn is not None else 0, 1 if leaky else 0)
    ptrs = [v.ctypes.data for v in vec] if vec else [None] * 3
    _lib.check_yolo(_lib.yolo_lib().gf_stage_yolo_conv(device, PRECISIONS[precision], shape, x.ctypes.data, w.ctypes.data,
                                                       bias.ctypes.data, *ptrs, out.ctypes.data))
    return out
