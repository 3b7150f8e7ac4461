"""The detector's TF32 mode without a GPU: the host emulation of cvt.rna.tf32.f32 the GPU tests rely on, the kernel's SASS
(HGMMA with TF32 operands, no spills), and the new C ABI in gf_b200.h and both libraries."""
import ctypes
import os
import re
import subprocess

import numpy as np
import pytest

from tf32_ref import rna_tf32

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "ground_fusion_b200")
NEW_SYMBOLS = ("gf_detector_set_precision", "gf_detector_get_precision", "gf_stage_yolo_conv")


def rna_float64(x):
    """The definition: the nearest value with an 11-bit significand (10 explicit bits) at x's binade, ties away from zero,
    computed in float64 (exact for every finite float32, subnormals included: their quantum is 2^-149 * 2^13)."""
    x = np.asarray(x, np.float32).astype(np.float64)
    out = np.empty_like(x)
    for i, v in enumerate(x.flat):
        if v == 0 or not np.isfinite(v):
            out.flat[i] = v
            continue
        e = max(int(np.floor(np.log2(abs(v)))), -126)
        q = 2.0 ** (e - 10)                       # spacing of 11-bit significands in this binade
        n = abs(v) / q                             # exact: v is a float32, q a power of two
        r = np.floor(n + 0.5)                      # ties away from zero on the magnitude
        out.flat[i] = np.copysign(r * q, v)
    return out


def _check(x):
    got = rna_tf32(x)
    with np.errstate(over="ignore"):
        want = rna_float64(x).astype(np.float32)      # exact, except that a carry past FLT_MAX is infinity in float32
    bad = got.view(np.uint32) != want.view(np.uint32)
    assert not bad.any(), (np.asarray(x)[bad][:5], got[bad][:5], want[bad][:5])
    assert np.all((rna_tf32(x).view(np.uint32) & 0x1FFF) == 0)


def test_rna_emulation_on_random_values():
    rng = np.random.default_rng(0)
    x = (rng.standard_normal(20000) * np.exp(rng.uniform(-40, 40, 20000))).astype(np.float32)
    _check(x)


def test_rna_emulation_on_ties_both_parities_and_signs():
    rng = np.random.default_rng(1)
    u = rng.integers(0x00800000, 0x7F000000, 4000, dtype=np.uint64).astype(np.uint32)
    u = (u & ~np.uint32(0x1FFF)) | np.uint32(0x1000)
    u[::2] |= np.uint32(0x80000000)
    x = u.view(np.float32)
    _check(x)
    # a tie rounds away from zero whatever the kept LSB: unlike ties-to-even on an even LSB
    even = np.array([0x3F801000], np.uint32).view(np.float32)
    assert rna_tf32(even).view(np.uint32)[0] == 0x3F802000
    assert rna_tf32(-even).view(np.uint32)[0] == 0xBF802000
    assert rna_tf32(np.array([0x3F800FFF], np.uint32).view(np.float32)).view(np.uint32)[0] == 0x3F800000


def test_rna_emulation_on_subnormals_and_carries():
    rng = np.random.default_rng(2)
    sub = rng.integers(1, 0x00800000, 4000, dtype=np.uint64).astype(np.uint32)
    sub[: 50] = (sub[: 50] & ~np.uint32(0x1FFF)) | np.uint32(0x1000)       # subnormal ties
    _check(sub.view(np.float32))
    _check(-sub.view(np.float32))
    # mantissa all ones above the rounding point: the carry moves into the exponent (and from the top subnormal to normal)
    carry = np.array([0x3FFFF000, 0x3FFFFFFF, 0x007FF000, 0x00FFF000, 0x7F7FF000, 0x00001000], np.uint32)
    _check(carry.view(np.float32))
    assert rna_tf32(np.array([0x3FFFF000], np.uint32).view(np.float32)).view(np.uint32)[0] == 0x40000000
    assert rna_tf32(np.array([0x007FF000], np.uint32).view(np.float32)).view(np.uint32)[0] == 0x00800000
    assert np.isinf(rna_tf32(np.array([0x7F7FF000], np.uint32).view(np.float32)))[0]
    _check(np.array([0.0, -0.0, 1.0, -2.5, np.float32(3.4e38)], np.float32))


def _built(name):
    p = os.path.join(PKG, name)
    if not os.path.exists(p):
        pytest.skip("%s not built" % name)
    return p


def test_tf32_kernel_issues_hgmma_with_tf32_operands():
    lib = _built("libgf_yolo.so")
    try:
        sass = subprocess.check_output(["cuobjdump", "-sass", lib], text=True, stderr=subprocess.STDOUT)
    except (OSError, subprocess.CalledProcessError) as e:
        pytest.skip("cuobjdump unavailable: %s" % e)
    funcs = re.split(r"\n\s+Function : ", sass)
    tf32 = [f for f in funcs if f.startswith("_ZN3gfy16k_yolo_conv_tf32")]
    assert len(tf32) == 1
    assert re.search(r"HGMMA\.64x64x8\.F32\.TF32", tf32[0])
    # the exact kernels stay off the tensor cores
    exact = [f for f in funcs if f.startswith("_ZN3gfy11k_yolo_conv")]
    assert len(exact) == 2 and not any("HGMMA" in f or "HMMA" in f for f in exact)


def test_no_detector_kernel_spills():
    log = os.path.join(ROOT, "build_ptxas_yolo.log")
    if not os.path.exists(log):
        pytest.skip("build_ptxas_yolo.log not written")
    text = open(log).read()
    entries = re.findall(r"Compiling entry function '(\w+)'.*?\n(.*?)\n(.*?)\n", text)
    assert any("k_yolo_conv_tf32" in e[0] for e in entries)
    for name, a, b in entries:
        for line in (a, b):
            m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", line)
            if m:
                assert m.group(1) == "0" and m.group(2) == "0", name


def test_header_declares_the_new_entry_points():
    h = open(os.path.join(ROOT, "include", "gf_b200.h")).read()
    assert "#define GF_DETECTOR_EXACT 0" in h and "#define GF_DETECTOR_TF32 1" in h
    for s in NEW_SYMBOLS:
        assert re.search(r"\bint %s\(" % s, h), s


@pytest.mark.parametrize("name", ["libgf_yolo.so", "libgf_b200.so"])
def test_both_libraries_export_the_new_entry_points(name):
    L = ctypes.CDLL(_built(name))
    for s in NEW_SYMBOLS:
        assert hasattr(L, s), s


def test_python_interface_refuses_unknown_precisions():
    from ground_fusion_b200.detector import PRECISIONS, YoloDetector, conv_stage
    assert PRECISIONS == {"exact": 0, "tf32": 1}
    with pytest.raises(ValueError):
        YoloDetector("none.cfg", "none.weights", precision="fp16")
    with pytest.raises(ValueError):
        conv_stage(np.zeros((1, 2, 2), np.float32), np.zeros((1, 1, 1, 1), np.float32), np.zeros(1, np.float32), precision="bf16")
