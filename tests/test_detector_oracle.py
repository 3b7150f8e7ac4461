"""The YOLO detector's host side and its oracle, without a GPU: the seeded .weights generator against darknet's load_weights,
the Python cfg parser against darknet's layer constructors for the six networks the reference ships, and the refusal of
networks outside them (by parse_cfg, and by gf_detector_create before it touches a device)."""
import ctypes
import os

import numpy as np
import pytest

from yolo_ref import CFGS, Darknet, cfg_at, cfg_path, conv_params_expected, oracle_available, write_weights

needs_oracle = pytest.mark.skipif(not oracle_available(), reason="darknet oracle not built (oracle/darknet.mk needs darknet's sources)")


@needs_oracle
@pytest.mark.parametrize("name", ["yolov2-tiny", "yolov2-voc", "yolov3"])
def test_weights_round_trip_through_darknet(name, tmp_path):
    cfg = cfg_at(name, str(tmp_path), 96, 96)
    w = write_weights(cfg, str(tmp_path / "w.weights"), seed=3)
    want = conv_params_expected(cfg, w)
    d = Darknet(cfg, w)
    try:
        assert len(want) == sum(L["type"] == "convolutional" for L in d.layers)
        for k, params in want.items():
            got = d.conv_params(k)
            assert sorted(got) == sorted(params)
            for key in params:
                assert np.array_equal(got[key], params[key]), (k, key)
    finally:
        d.close()


@needs_oracle
@pytest.mark.parametrize("size", [None, (160, 160), (320, 192)])
@pytest.mark.parametrize("name", CFGS)
def test_cfg_parser_matches_darknet(name, size, tmp_path):
    from ground_fusion_b200.detector import parse_cfg
    cfg = cfg_path(name) if size is None else cfg_at(name, str(tmp_path), *size)
    net, layers = parse_cfg(cfg)
    d = Darknet(cfg)
    try:
        assert (net["w"], net["h"], net["c"]) == (d.w, d.h, d.c)
        assert len(layers) == d.n
        for L, D in zip(layers, d.layers):
            assert L["type"] == D["type"] or (L["type"], D["type"]) == ("upsample", "none")   # darknet has no name for it
            for k in ("out_w", "out_h", "out_c", "outputs"):
                assert L[k] == D[k], (L["type"], k)
            if L["type"] == "convolutional":
                for k in ("n", "size", "stride", "pad", "batch_normalize"):
                    assert L[k] == D[k], k
                assert L["n"] * L["c"] * L["size"] ** 2 == D["nweights"]
    finally:
        d.close()


def _variant(tmp_path, name, old, new):
    text = open(cfg_path(name)).read()
    assert old in text
    p = tmp_path / ("v_" + name + ".cfg")
    p.write_text(text.replace(old, new, 1))
    return str(p)


REFUSED = [
    ("yolov2-tiny", "[maxpool]", "[avgpool]", "unsupported layer type [avgpool]"),
    ("yolov2-tiny", "activation=leaky", "activation=relu", "unsupported activation 'relu'"),
    ("yolov2-tiny", "activation=leaky", "activation=logistic", "unsupported activation 'logistic'"),
    ("yolov2-tiny", "filters=16", "filters=16\ngroups=2", "groups"),
    ("yolov2-tiny", "filters=16", "filters=16\nxnor=1", "xnor"),
    ("yolov2", "[reorg]\nstride=2", "[reorg]\nstride=2\nreverse=1", "reverse"),
    ("yolov2-tiny", "coords=4", "coords=5", "coords"),
    ("yolov2-tiny", "softmax=1", "softmax=1\ntree=data/9k.tree", "softmax trees"),
    ("yolov3", "stride=2\n\n[route]", "stride=-2\n\n[route]", "reverse (negative stride) upsample"),
    ("yolov3", "[net]", "[net]\nchannels=1", "channels"),
]


@pytest.mark.parametrize("name,old,new,msg", REFUSED)
def test_unsupported_networks_are_refused(name, old, new, msg, tmp_path):
    """gf_detector_create reads the files before it selects a device, so the refusal (GF_ERR_UNSUPPORTED and a message naming
    what is unsupported) shows on any machine; an empty weights file does not matter, the cfg is refused first."""
    from ground_fusion_b200 import _lib
    cfg = _variant(tmp_path, name, old, new)
    weights = tmp_path / "empty.weights"
    weights.write_bytes(b"")
    L = _lib.yolo_lib()
    h = ctypes.c_void_p()
    rc = L.gf_detector_create(ctypes.byref(h), 0, cfg.encode(), str(weights).encode(), ctypes.c_float(0.3))
    assert rc == -5, (rc, L.gf_detector_last_error())          # GF_ERR_UNSUPPORTED
    assert msg in L.gf_detector_last_error().decode()
    assert not h.value


def test_python_parser_refuses_unknown_layers(tmp_path):
    from ground_fusion_b200.detector import parse_cfg
    with pytest.raises(ValueError, match="avgpool"):
        parse_cfg(_variant(tmp_path, "yolov2-tiny", "[maxpool]", "[avgpool]"))


def test_short_weights_are_refused(tmp_path):
    from ground_fusion_b200 import _lib
    cfg = cfg_at("yolov2-tiny", str(tmp_path), 96, 96)
    w = write_weights(cfg, str(tmp_path / "w.weights"))
    data = open(w, "rb").read()
    short = tmp_path / "short.weights"
    short.write_bytes(data[:-4])
    L = _lib.yolo_lib()
    h = ctypes.c_void_p()
    rc = L.gf_detector_create(ctypes.byref(h), 0, cfg.encode(), str(short).encode(), ctypes.c_float(0.3))
    assert rc == -1 and b"ends inside layer" in L.gf_detector_last_error()


def test_extraction_rules():
    """darknet_ros's extraction: clamped to the frame, > 1 % of it, one box per class with a non-zero probability, grouped by
    class, corners by int truncation; more than 100 boxes publish nothing."""
    from yolo_ref import extract
    bbox = np.array([[0.5, 0.5, 0.2, 0.2], [0.05, 0.95, 0.3, 0.3], [0.5, 0.5, 0.005, 0.5]], np.float32)
    prob = np.zeros((3, 3), np.float32)
    prob[0, 2] = 0.9; prob[0, 0] = 0.4; prob[1, 1] = 0.5; prob[2, 0] = 0.8
    b, c, p = extract(bbox, prob, 640, 480)
    assert c == [0, 1, 2]
    assert b[0] == b[2] == (255, 191, 384, 288)       # (0.5f - 0.1f) * 640 rounds to just under 256 and truncates
    assert b[1] == (0, 383, 128, 480)
    many = np.tile(np.array([[0.5, 0.5, 0.2, 0.2]], np.float32), (101, 1))
    assert extract(many, np.full((101, 1), 0.5, np.float32), 640, 480) == ([], [], [])
    assert len(extract(many[:100], np.full((100, 1), 0.5, np.float32), 640, 480)[0]) == 100
