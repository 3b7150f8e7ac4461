"""Network sizes the detector refuses, without a GPU.  yolov2 and yolov3 (and their VOC cfgs) only work at multiples of 32: at
another [net] size a [route] joins maps of different sizes (a floored stride-2 layer on one side, an upsample or a floored
reorg on the other), and darknet's parse_route then zeroes the route's out_w / out_h / out_c, so every later layer of the
network sees an empty input.  gf_detector_create refuses such a network by name (before it touches a device): at the [reorg]
whose input its stride does not divide, or at the [route] whose inputs differ in size, whichever comes first."""
import pytest

from yolo_ref import Darknet, cfg_at, oracle_available

NETS = ("yolov2", "yolov2-voc", "yolov3", "yolov3-voc")
SIZES = ((200, 136), (416, 400))          # neither a multiple of 32 in both directions


def first_bad_route(layers):
    """The index of the first [route] whose inputs differ in size (layers as parse_cfg gives them), or None."""
    for i, L in enumerate(layers):
        if L["type"] == "route" and len({(layers[k]["out_w"], layers[k]["out_h"]) for k in L["inputs"]}) > 1:
            return i
    return None


def expected_refusal(layers):
    """gf_detector_create's error text for these layers, from their arithmetic: the first [reorg] whose stride does not divide
    its input, or the first [route] whose inputs differ in size; None if neither occurs."""
    r = first_bad_route(layers)
    for i, L in enumerate(layers):
        if L["type"] == "reorg" and (L["w"] % L["stride"] or L["h"] % L["stride"]):
            return "[reorg] layer %d: reorg stride must divide the input" % i
        if i == r:
            return "[route] layer %d: route inputs of different sizes are not supported" % i
    return None


@pytest.mark.parametrize("size", SIZES, ids=["%dx%d" % s for s in SIZES])
@pytest.mark.parametrize("name", NETS)
def test_sizes_off_multiples_of_32_are_refused_by_name(name, size, tmp_path):
    from ground_fusion_b200._lib import GfError
    from ground_fusion_b200.detector import YoloDetector, parse_cfg
    cfg = cfg_at(name, str(tmp_path), *size)
    _, layers = parse_cfg(cfg)
    assert first_bad_route(layers) is not None
    msg = expected_refusal(layers)
    assert msg.startswith("[reorg]" if name.startswith("yolov2") else "[route]")
    weights = tmp_path / "empty.weights"
    weights.write_bytes(b"")                     # the cfg is refused before the weights are read
    with pytest.raises(GfError) as e:
        YoloDetector(cfg, str(weights))
    assert str(e.value).endswith(msg), str(e.value)
    assert "error -5:" in str(e.value)           # GF_ERR_UNSUPPORTED


@pytest.mark.skipif(not oracle_available(), reason="darknet oracle not built (oracle/darknet.mk needs darknet's sources)")
@pytest.mark.parametrize("size", SIZES, ids=["%dx%d" % s for s in SIZES])
@pytest.mark.parametrize("name", NETS)
def test_darknet_zeroes_the_route_at_these_sizes(name, size, tmp_path):
    """darknet's own shapes: every layer before the first mismatched [route] as parse_cfg gives it, and the route itself with
    out_w = out_h = out_c = 0.  The whole cfg cannot be loaded in this process: the [convolutional] after the route calls
    darknet's error() on its empty input, which asserts and aborts.  So darknet loads the cfg cut after the route, and the
    layer that would stop it is checked from the cfg."""
    from ground_fusion_b200.detector import parse_cfg
    cfg = cfg_at(name, str(tmp_path), *size)
    _, layers = parse_cfg(cfg)
    r = first_bad_route(layers)
    assert layers[r + 1]["type"] == "convolutional"
    lines = open(cfg).read().splitlines()
    heads = [j for j, ln in enumerate(lines) if ln.strip().startswith("[")]       # [net], then layer k at heads[k + 1]
    cut = tmp_path / "cut.cfg"
    cut.write_text("\n".join(lines[:heads[r + 2]]) + "\n")
    d = Darknet(str(cut))
    try:
        assert d.n == r + 1
        for k in range(r):
            assert d.layers[k]["type"] == layers[k]["type"] or (layers[k]["type"], d.layers[k]["type"]) == ("upsample", "none")
            assert [d.layers[k][f] for f in ("out_w", "out_h", "out_c")] == [layers[k][f] for f in ("out_w", "out_h", "out_c")], k
        R = d.layers[r]
        assert R["type"] == "route" and (R["out_w"], R["out_h"], R["out_c"]) == (0, 0, 0), R
    finally:
        d.close()
