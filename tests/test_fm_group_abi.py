"""CPU checks of gf_fm_window_group's C ABI: every entry point the header declares is exported by the library with the ctypes
prototype the Python layer uses (argument count as declared), and the group limit matches the tracker group's."""
import os
import re
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared():
    src = open(os.path.join(ROOT, "include", "gf_b200.h")).read()
    out = {}
    for m in re.finditer(r"^(?:int|void) (gf_fm_window_group_\w+)\(([^;]*)\);", src, re.M):
        out[m.group(1)] = len([a for a in m.group(2).split(",") if a.strip()])
    return out, src


def test_group_entry_points_have_prototypes():
    from ground_fusion_b200 import _lib
    L = _lib.lib()
    decl, _ = _declared()
    assert len(decl) == 15, sorted(decl)
    for name, nargs in decl.items():
        fn = getattr(L, name)
        assert fn.argtypes is not None and len(fn.argtypes) == nargs, name


def test_group_limit_equals_tracker_group_limit():
    from ground_fusion_b200 import _lib
    _, src = _declared()
    fm = int(re.search(r"#define GF_FM_WINDOW_GROUP_MAX (\d+)", src).group(1))
    tr = int(re.search(r"#define GF_TRACKER_GROUP_MAX (\d+)", src).group(1))
    assert fm == tr == _lib.FM_WINDOW_GROUP_MAX
    ops = [int(re.search(r"#define GF_FM_REMOVE_%s (\d+)" % n, src).group(1)) for n in ("NONE", "BACK_SHIFT_DEPTH", "BACK", "FRONT")]
    assert ops == [_lib.FM_REMOVE_NONE, _lib.FM_REMOVE_BACK_SHIFT_DEPTH, _lib.FM_REMOVE_BACK, _lib.FM_REMOVE_FRONT]


def test_harness_with_the_group_bench_compiles_and_links():
    subprocess.check_call(["make", "-s", "-C", os.path.join(ROOT, "adaptor")])
    harness = os.path.join(ROOT, "adaptor", "_build", "harness")
    syms = subprocess.check_output(["nm", "-D", "--undefined-only", harness]).decode()
    for s in ("create", "destroy", "add_frame", "triangulate", "fill_problem", "set_depth", "remove", "remove_failures", "remove_ids",
              "outliers", "predict_next", "last_device_ms"):
        assert (" U gf_fm_window_group_" + s + "\n") in syms, s
    usage = subprocess.run([harness], capture_output=True, text=True)
    assert usage.returncode == 2 and "fm-group-bench" in usage.stderr
