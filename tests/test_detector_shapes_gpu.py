"""The YOLO detector at non-square and odd [net] sizes against darknet's CPU build (tests/yolo_ref.py).

Every other detector test builds square networks, where a w / h swap anywhere (the letterbox, the conv's pixel split, maxpool,
reorg, upsample, the TF32 gather table, the box decoding, correct_boxes) changes nothing.  Here:
- the six networks at 320 x 192 and 192 x 320 (10 x 6 / 6 x 10 heads, reorg 20 x 12 -> 10 x 6, upsample and route on
  non-square maps); yolov2-tiny and yolov2-tiny-voc also at 200 x 136 (odd inputs to the stride-2 maxpools: 25 -> 13, 13 -> 7,
  17 -> 9, 9 -> 5, and the stride-1 pool at 7 x 5), and at 32 x 256 and 256 x 32 (a head grid one cell wide / one cell tall);
- exact mode bit for bit with darknet: the letterboxed input, every layer's output (on one frame; the last layer on the
  others) and the published boxes, class ids and probabilities at two thresholds, on landscape, portrait, exact-aspect,
  row-padded 641 x 481 and 1 x 1 frames;
- the letterbox stage alone at seven net sizes and eight frames;
- TF32 mode: every convolution within DESIGN.md's bound, the dyadic exactness check on every new convolution shape, and the
  TF32 heads decoded as darknet decodes them;
- detect_batch on mixed frame sizes, each member equal to detect alone (and, exact, to darknet).
A darknet forward of yolov2 / yolov3 takes seconds on the CPU, so each frame's darknet result is computed once per network and
size and shared by the tests that need it.  Sizes that are not multiples of 32 for yolov2 / yolov3 are refused:
test_detector_shapes.py."""
import tempfile

import numpy as np
import pytest

from test_detector_batch_gpu import assert_bits, assert_same_result
from test_detector_gpu import random_bgr, synth_bgr
from test_detector_tf32_gpu import SHAPES
from tf32_ref import check_dyadic_operands, conv_shapes, detect_from_heads, heads_oracle_available, layer_bound_check
from yolo_ref import CFGS, Darknet, cfg_at, extract, oracle_available, write_weights

pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(not oracle_available(), reason="darknet oracle not built (oracle/darknet.mk needs darknet's sources)")]

WIDE, TALL = (320, 192), (192, 320)
ODD, ONE_WIDE, ONE_TALL = (200, 136), (32, 256), (256, 32)
TINY = ("yolov2-tiny", "yolov2-tiny-voc")
THRESHOLDS = (0.3, 0.7)
CASES = [(n, s) for n in CFGS for s in (WIDE, TALL)] + [(n, s) for n in TINY for s in (ODD, ONE_WIDE, ONE_TALL)]
ALL_FRAMES = ("640x480", "480x640", "aspect", "641x481", "1x1")
BATCH_FRAMES = ("640x480", "480x640", "aspect", "1x1")


def _id(s):
    return "%dx%d" % s


def frame(key, nw, nh):
    """The test frames: synthetic 640 x 480, random portrait 480 x 640, random at twice the net size (the net's exact aspect:
    (float)nw / w == (float)nh / h, the tie correct_boxes and the letterbox send to their else branch), the synthetic frame
    padded to 641 x 481 as a view of rows 654 pixels apart, and 1 x 1."""
    if key == "640x480":
        return synth_bgr(0)
    if key == "480x640":
        return random_bgr(3, 480, 640)
    if key == "aspect":
        return random_bgr(7, 2 * nw, 2 * nh)
    if key == "641x481":
        rows = np.zeros((481, 654, 3), np.uint8)
        rows[:, :641] = np.pad(synth_bgr(5), ((0, 1), (0, 1), (0, 0)), mode="edge")
        return rows[:, :641]
    assert key == "1x1"
    return random_bgr(4, 16, 16)[:1, :1].copy()


def frames_for(name, size):
    """One or two darknet forwards per size for the four large networks: the frame checked layer by layer first."""
    if name in TINY:
        return ALL_FRAMES
    return ("640x480", "480x640") if size == WIDE else ("480x640", "640x480")


class Oracle:
    """The networks' files and darknet on them, kept for the module: each (network, size, frame) is run through darknet once,
    keeping its letterboxed input, last layer and published results at THRESHOLDS; layers=True also returns every layer's
    output of that run (not kept)."""

    def __init__(self, d):
        self.d = d
        self._files, self._nets, self._runs = {}, {}, {}

    def files(self, name, size):
        if (name, size) not in self._files:
            cfg = cfg_at(name, self.d, *size)
            self._files[name, size] = (cfg, write_weights(cfg, "%s/%s_%dx%d.weights" % (self.d, name, size[0], size[1]), seed=1))
        return self._files[name, size]

    def darknet(self, name, size):
        if (name, size) not in self._nets:
            self._nets[name, size] = Darknet(*self.files(name, size))
        return self._nets[name, size]

    def run(self, name, size, key, layers=False):
        got = self._runs.get((name, size, key))
        if got is not None and not layers:
            return got
        ref = self.darknet(name, size)
        bgr = frame(key, *size)
        x = ref.forward(bgr)
        got = {"input": x, "last": ref.layer_output(ref.n - 1), "boxes": {}}
        for t in THRESHOLDS:
            bbox, _, prob = ref.detections(bgr.shape[1], bgr.shape[0], t)
            b, c, p = extract(bbox, prob, bgr.shape[1], bgr.shape[0])
            got["boxes"][t] = (np.array(b, np.int64).reshape(-1, 4), np.array(c, np.int32), np.array(p, np.float32))
        self._runs[name, size, key] = got
        if layers:
            return dict(got, layers=[ref.layer_output(k) for k in range(ref.n)])
        return got

    def close(self):
        for r in self._nets.values():
            r.close()


@pytest.fixture(scope="module")
def oracle(tmp_path_factory):
    o = Oracle(str(tmp_path_factory.mktemp("yolo_shapes")))
    try:
        yield o
    finally:
        o.close()


@pytest.mark.parametrize("name,size", CASES, ids=["%s-%s" % (n, _id(s)) for n, s in CASES])
def test_exact_mode_matches_darknet(name, size, oracle):
    """The letterboxed input, every layer (first frame) or the last layer (the others), and the boxes at both thresholds."""
    from ground_fusion_b200.detector import YoloDetector
    cfg, w = oracle.files(name, size)
    dets = {t: YoloDetector(cfg, w, thresh=t) for t in THRESHOLDS}
    counts = {}
    try:
        det = dets[THRESHOLDS[0]]
        assert (det.net_w, det.net_h) == size
        for j, key in enumerate(frames_for(name, size)):
            want = oracle.run(name, size, key, layers=j == 0)
            bgr = frame(key, *size)
            for t in THRESHOLDS:
                got = dets[t].detect(bgr)
                assert_same_result(got, want["boxes"][t], "%s thresh %.1f" % (key, t))
                counts[key, t] = len(got[0])
            assert_bits(det.input_image(), want["input"], "%s letterboxed input" % key)
            if j == 0:
                for k, ref in enumerate(want["layers"]):
                    assert_bits(det.layer_output(k), ref, "%s layer %d" % (key, k))
            else:
                assert_bits(det.layer_output(det.n_layers - 1), want["last"], "%s last layer" % key)
    finally:
        for d in dets.values():
            d.close()
    if name in ("yolov2-tiny", "yolov3") and size in (WIDE, TALL):
        assert any(n > 1 for n in counts.values()), counts     # NMS and the extraction run on a non-square grid


LETTERBOX_NETS = (WIDE, TALL, ODD, ONE_WIDE, ONE_TALL, (416, 416), (33, 65))


@pytest.mark.parametrize("size", LETTERBOX_NETS, ids=[_id(s) for s in LETTERBOX_NETS])
def test_letterbox_stage_matches_darknet(size, tmp_path):
    """gf_stage_letterbox against darknet's letterbox_image at the net size, bit for bit, on frames of both orientations,
    tiny and odd frames, a row-padded view and the net's exact aspect."""
    from ground_fusion_b200.detector import letterbox
    nw, nh = size
    ref = Darknet(cfg_at("yolov2-tiny", str(tmp_path), nw, nh))
    try:
        assert (ref.w, ref.h) == size
        for (fw, fh) in ((640, 480), (480, 640), (1280, 720), (641, 481), (100, 37), (2, 3), (1, 1), (2 * nw, 2 * nh)):
            bgr = random_bgr(fw * 7 + fh, fw + 16, fh + 16)[:fh, :fw]       # a view with padded rows
            got = letterbox(bgr, nw, nh)
            assert_bits(got, ref.letterbox(bgr), "%dx%d frame" % (fw, fh))
    finally:
        ref.close()


TF32_CASES = [(n, s) for n in CFGS for s in (WIDE, TALL)]


@pytest.mark.parametrize("name,size", TF32_CASES, ids=["%s-%s" % (n, _id(s)) for n, s in TF32_CASES])
def test_tf32_every_convolution_within_the_error_bound(name, size, oracle):
    from ground_fusion_b200.detector import YoloDetector
    cfg, w = oracle.files(name, size)
    det = YoloDetector(cfg, w, thresh=0.3, precision="tf32")
    try:
        det.detect(synth_bgr(0))
        worst = layer_bound_check(det, cfg, w)
    finally:
        det.close()
    print("%s at %s: largest error / bound %.4f" % (name, _id(size), worst))


def _new_shapes():
    seen = set()
    with tempfile.TemporaryDirectory() as d:
        for name, size in CASES:
            seen.update(conv_shapes(cfg_at(name, d, *size)))
    return sorted(seen - set(SHAPES))


NEW_SHAPES = _new_shapes()


@pytest.mark.parametrize("shape", NEW_SHAPES, ids=["C%d_H%d_W%d_M%d_s%d_st%d_p%d" % s for s in NEW_SHAPES])
def test_tf32_dyadic_operands_give_the_exact_modes_bits(shape):
    check_dyadic_operands(shape)


@pytest.mark.skipif(not heads_oracle_available(), reason="darknet heads oracle not built")
def test_decoding_of_the_tf32_heads_matches_darknet(oracle):
    """yolov3 at 320 x 192: the TF32 mode's boxes are darknet's decoding, NMS and extraction of its own [yolo] outputs."""
    from ground_fusion_b200.detector import YoloDetector
    cfg, w = oracle.files("yolov3", WIDE)
    ref = oracle.darknet("yolov3", WIDE)
    heads = [k for k, L in enumerate(ref.layers) if L["type"] == "yolo"]
    published = 0
    for thresh in THRESHOLDS:
        det = YoloDetector(cfg, w, thresh=thresh, precision="tf32")
        try:
            for key in BATCH_FRAMES:
                bgr = frame(key, *WIDE)
                got = det.detect(bgr)
                bbox, _, prob = detect_from_heads(ref, {i: det.layer_output(i) for i in heads}, bgr.shape[1], bgr.shape[0], thresh)
                b, c, p = extract(bbox, prob, bgr.shape[1], bgr.shape[0])
                assert_same_result(got, (np.array(b, np.int64).reshape(-1, 4), np.array(c, np.int32), np.array(p, np.float32)),
                                   "%s thresh %.1f" % (key, thresh))
                published += len(got[0])
        finally:
            det.close()
    assert published > 0


BATCH_CASES = [("yolov2-tiny", ODD), ("yolov3", WIDE)]


@pytest.mark.parametrize("precision", ("exact", "tf32"))
@pytest.mark.parametrize("name,size", BATCH_CASES, ids=["%s-%s" % (n, _id(s)) for n, s in BATCH_CASES])
def test_batch_of_mixed_frames_equals_single_detects(name, size, precision, oracle):
    """detect_batch on a landscape, a portrait, an exact-aspect and a 1 x 1 frame: each member's boxes, letterboxed input and
    last layer equal detect on that frame alone, and in exact mode darknet's."""
    from ground_fusion_b200.detector import YoloDetector
    cfg, w = oracle.files(name, size)
    frames = [frame(k, *size) for k in BATCH_FRAMES]
    bat = YoloDetector(cfg, w, thresh=THRESHOLDS[0], precision=precision)
    one = YoloDetector(cfg, w, thresh=THRESHOLDS[0], precision=precision)
    try:
        bat.set_max_batch(len(frames))
        got = bat.detect_batch(frames)
        assert len(got) == len(frames)
        last = one.n_layers - 1
        for i, (key, bgr) in enumerate(zip(BATCH_FRAMES, frames)):
            want = one.detect(bgr)
            assert_same_result(got[i], want, "member %d (%s)" % (i, key))
            assert_bits(bat.member_layer_output(i, -1), one.input_image(), "member %d input" % i)
            assert_bits(bat.member_layer_output(i, last), one.layer_output(last), "member %d last layer" % i)
            if precision == "exact":
                ref = oracle.run(name, size, key)
                assert_same_result(got[i], ref["boxes"][THRESHOLDS[0]], "member %d (%s) against darknet" % (i, key))
                assert_bits(bat.member_layer_output(i, -1), ref["input"], "member %d input against darknet" % i)
                assert_bits(bat.member_layer_output(i, last), ref["last"], "member %d last layer against darknet" % i)
    finally:
        bat.close()
        one.close()
