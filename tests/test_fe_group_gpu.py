"""GPU tests of gf_tracker_group (TrackerGroup): K trackers stepped in lockstep by one set of launches per step must give,
member by member, byte for byte, what the same trackers give on their own (trackBatch / trackImage / trackImagebox).
Run with -m gpu on an H100."""
import ctypes

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

_FRAMES = {}


def frames(seed, n, w=640, h=480, no_depth=()):
    """n frames (t, gray, depth or None) of SyntheticStream(seed) at w x h; frames whose index is in no_depth have no depth image."""
    from ground_fusion_b200.synth import SyntheticStream
    key = (seed, w, h)
    if key not in _FRAMES or len(_FRAMES[key]) < n:
        st = SyntheticStream(seed=seed, width=w, height=h)
        _FRAMES[key] = [tuple(np.ascontiguousarray(x) if isinstance(x, np.ndarray) else x for x in st.frame(k)) for k in range(n)]
    return [(t, g, (None if k in no_depth else d)) for k, (t, g, d) in enumerate(_FRAMES[key][:n])]


def params8(w, fx_scale=1.0):
    from ground_fusion_b200.synth import idc_params8
    p, sc = idc_params8(), w / 640.0
    return [p[0] * sc * fx_scale, p[1] * sc * fx_scale, p[2] * sc, p[3] * sc] + p[4:]


class Ptrs:
    """Frame addresses for the batch calls: the host arrays themselves, or copies resident on the device (kept alive here)."""

    def __init__(self, on_device):
        self.on_device, self.keep = on_device, []

    def __call__(self, fr):
        if not self.on_device:
            return [g.ctypes.data for _, g, _ in fr], [(d.ctypes.data if d is not None else 0) for _, _, d in fr]
        import torch
        gs = [torch.from_numpy(g).cuda() for _, g, _ in fr]
        ds = [(torch.from_numpy(d.view(np.int16)).cuda() if d is not None else None) for _, _, d in fr]
        self.keep.append((gs, ds))
        torch.cuda.synchronize()
        return [x.data_ptr() for x in gs], [(x.data_ptr() if x is not None else 0) for x in ds]


@pytest.fixture(params=["tma", "no-tma"])
def lk_staging(request, monkeypatch):
    """make_lk_maps reads GF_LK_NO_TMA when a tracker is created: with it the LK windows are staged by ordinary loads."""
    if request.param == "no-tma":
        monkeypatch.setenv("GF_LK_NO_TMA", "1")
    else:
        monkeypatch.delenv("GF_LK_NO_TMA", raising=False)
    return request.param


def same(want, got, what):
    """Per-frame results (obs, status, info[, in_box]) byte for byte."""
    assert len(want) == len(got), what
    for k, (a, b) in enumerate(zip(want, got)):
        assert a[2] == b[2], "%s frame %d: info" % (what, k)
        assert np.array_equal(a[1], b[1]), "%s frame %d: status" % (what, k)
        assert a[0].tobytes() == b[0].tobytes(), "%s frame %d: obs" % (what, k)
        if len(a) > 3:
            assert np.array_equal(a[3], b[3]), "%s frame %d: in_box" % (what, k)


def pair(S, w=640, h=480, max_cnt=150, min_dist=30, fx_scale=None, equalize=False):
    """S reference trackers and S group members with the same configuration (member i's intrinsics scaled by fx_scale[i])."""
    from ground_fusion_b200.feature_tracker import FeatureTracker
    fx = fx_scale or [1.0] * S
    mk = lambda i: FeatureTracker(w, h, params8(w, fx[i]), max_cnt, min_dist, 1, 1, equalize=equalize)   # noqa: E731
    return [mk(i) for i in range(S)], [mk(i) for i in range(S)]


def close(*lists):
    for L in lists:
        for x in L:
            x.close()


def batch_compare(S, n, on_device, w=640, h=480, max_cnt=150, min_dist=30, equalize=False, seed0=40, mixed=False):
    """n steps of S members through TrackerGroup.trackBatch against S trackBatch calls on separate trackers.  mixed: different
    intrinsics, member 1 without depth images on some frames, member 2 with a pending prediction when the group starts."""
    from ground_fusion_b200.feature_tracker import TrackerGroup
    ref, mem = pair(S, w, h, max_cnt, min_dist, [1.0 + 0.05 * (i % 3) for i in range(S)] if mixed else None, equalize)
    fr = [frames(seed0 + i, n + 2, w, h, no_depth=(3, 4, 8) if (mixed and i == 1) else ()) for i in range(S)]
    for i in range(S):
        for t, g, d in fr[i][:2]:
            o = ref[i].trackImageRaw(t, g, d)
            mem[i].trackImageRaw(t, g, d)
        if mixed and i == 2:
            pred = {int(x["id"]): (x["v"][0] * 2.0, x["v"][1] * 2.0, 2.0) for x in o[::2]}
            ref[i].setPrediction(pred)
            mem[i].setPrediction(pred)
    P = Ptrs(on_device)
    ptr = [P(fr[i][2:]) for i in range(S)]
    times = [[t for t, _, _ in fr[i][2:]] for i in range(S)]
    want = [ref[i].trackBatch(times[i], *ptr[i], on_device=on_device) for i in range(S)]
    G = TrackerGroup(mem)
    got = G.trackBatch(times, [p[0] for p in ptr], [p[1] for p in ptr], on_device=on_device)
    for i in range(S):
        same(want[i], got[i], "member %d" % i)
        assert mem[i].last_info == ref[i].last_info
    G.close()
    close(ref, mem)
    return got


@pytest.mark.parametrize("on_device", [False, True])
def test_three_mixed_members(on_device, lk_staging):
    got = batch_compare(3, 9, on_device, mixed=True)
    assert sum(len(o) for o, _, _ in got[0]) > 500


@pytest.mark.parametrize("on_device", [False, True])
def test_group_of_one(on_device, lk_staging):
    batch_compare(1, 6, on_device)


@pytest.mark.parametrize("on_device", [False, True])
def test_interleaved_direct_use(on_device, lk_staging):
    """Group steps, then trackImage on member 0, removeOutliers on member 1 and a prediction on member 2 bad enough that fewer
    than 10 points succeed (the 3-level fallback), then more group steps: the members end at different frame counters mod 3."""
    from ground_fusion_b200.feature_tracker import TrackerGroup
    S = 3
    ref, mem = pair(S, fx_scale=[1.0, 1.03, 0.97])
    twin = pair(1, fx_scale=[0.97])[0][0]           # member 2's stream without the prediction
    fr = [frames(60 + i, 12) for i in range(S)]
    P = Ptrs(on_device)
    G = TrackerGroup(mem)

    def steps(k0, k1, ks):
        ptr = [P([fr[i][k] for k in ks[i]]) for i in range(S)]
        times = [[fr[i][k][0] for k in ks[i]] for i in range(S)]
        want = [ref[i].trackBatch(times[i], *ptr[i], on_device=on_device) for i in range(S)]
        got = G.trackBatch(times, [p[0] for p in ptr], [p[1] for p in ptr], on_device=on_device)
        for i in range(S):
            same(want[i], got[i], "member %d, steps %d-%d" % (i, k0, k1))
        return got

    got = steps(0, 4, [range(0, 4)] * S)
    t, g, d = fr[0][4]
    o1 = ref[0].trackImageRaw(t, g, d)
    o2 = mem[0].trackImageRaw(t, g, d)
    assert o1.tobytes() == o2.tobytes()
    ids = [int(x["id"]) for x in got[1][-1][0][::3]]
    ref[1].removeOutliers(ids)
    mem[1].removeOutliers(ids)
    # every feature of member 2 is predicted at (1.5, 0, 1), which projects about 690 px left of the image: the prediction
    # pass finds no point (fewer than 10 successes) and k_track runs its own 3-level LK, so the frame is exactly what the
    # twin without a prediction tracks
    bad = {int(x["id"]): (1.5, 0.0, 1.0) for x in got[2][-1][0]}
    ref[2].setPrediction(bad)
    mem[2].setPrediction(bad)
    for t, g, d in fr[2][:4]:
        twin.trackImageRaw(t, g, d)
    got = steps(5, 11, [range(5, 11), range(4, 10), range(4, 10)])
    o, st, info = got[2][0]
    assert info["n_prev"] > 10 and o.tobytes() == twin.trackImageRaw(*fr[2][4]).tobytes()
    assert np.array_equal(st, twin.last_status) and info == twin.last_info
    G.close()
    close(ref, mem, [twin])


@pytest.mark.parametrize("on_device", [False, True])
def test_two_steps_in_flight(on_device, lk_staging):
    """submit / wait with two steps in flight equals trackBatch on separate trackers."""
    from ground_fusion_b200.feature_tracker import TrackerGroup
    S, n = 4, 7
    ref, mem = pair(S)
    fr = [frames(70 + i, n, no_depth=(2,) if i == 3 else ()) for i in range(S)]
    P = Ptrs(on_device)
    ptr = [P(fr[i]) for i in range(S)]
    want = [ref[i].trackBatch([t for t, _, _ in fr[i]], *ptr[i], on_device=on_device) for i in range(S)]
    G = TrackerGroup(mem)
    got = [[] for _ in range(S)]

    def collect():
        for i, r in enumerate(G.wait()):
            got[i].append(r[:3])
    for k in range(n):
        G.submit([fr[i][k][0] for i in range(S)], [ptr[i][0][k] for i in range(S)], [ptr[i][1][k] for i in range(S)], on_device=on_device)
        if k >= 1:
            collect()
    collect()
    for i in range(S):
        same(want[i], got[i], "member %d" % i)
    G.close()
    close(ref, mem)


def _boxes(rng, m, w=640, h=480):
    x0, y0 = rng.integers(-20, w, m), rng.integers(-20, h, m)
    return np.stack([x0, y0, x0 + rng.integers(-10, 200, m), y0 + rng.integers(-10, 160, m)], 1).astype(np.int64)


@pytest.mark.parametrize("on_device", [False, True])
def test_boxes_per_member_and_step(on_device, lk_staging):
    """Per-member, per-step detections (none, a few, GF_MAX_BOXES) give trackImagebox's in_box flags."""
    from ground_fusion_b200.feature_tracker import TrackerGroup
    S, n = 3, 6
    rng = np.random.default_rng(5)
    ref, mem = pair(S)
    fr = [frames(80 + i, n) for i in range(S)]
    boxes = [[_boxes(rng, [0, 3, 100, 1, 0, 7][(k + i) % 6]) for k in range(n)] for i in range(S)]
    want = [[ref[i].trackImageboxRaw(t, boxes[i][k], g, d) for k, (t, g, d) in enumerate(fr[i])] for i in range(S)]
    P = Ptrs(on_device)
    ptr = [P(fr[i]) for i in range(S)]
    G = TrackerGroup(mem)
    got = G.trackBatch([[t for t, _, _ in fr[i]] for i in range(S)], [p[0] for p in ptr], [p[1] for p in ptr], on_device=on_device, boxes=boxes)
    for i in range(S):
        for k in range(n):
            o, _, _, ib = got[i][k]
            assert o.tobytes() == want[i][k][0].tobytes() and np.array_equal(ib, want[i][k][1]), "member %d step %d" % (i, k)
        assert any(ib.any() for _, _, _, ib in got[i])
    G.close()
    close(ref, mem)


@pytest.mark.parametrize("on_device", [False, True])
def test_equalize(on_device, lk_staging):
    batch_compare(3, 6, on_device, equalize=True, seed0=90)


@pytest.mark.parametrize("geom", ["C3", "1280x720_500", "max_cnt_1000", "narrow_600"])
@pytest.mark.parametrize("on_device", [False, True])
def test_other_sizes(on_device, geom, lk_staging):
    w, h, mc, md = {"C3": (640, 480, 300, 20), "1280x720_500": (1280, 720, 500, 25), "max_cnt_1000": (640, 480, 1000, 10),
                    "narrow_600": (600, 480, 150, 30)}[geom]
    got = batch_compare(2, 5, on_device, w, h, mc, md, seed0=100)
    assert max(len(o) for o, _, _ in got[0]) > min(mc // 2, 100)


@pytest.mark.parametrize("on_device", [False, True])
def test_k32(on_device, lk_staging):
    batch_compare(32, 6, on_device, seed0=200)


def test_launch_count_does_not_grow_with_k():
    """Per step: the single tracker's per-frame launch count, plus the prediction launch when any member has a prediction."""
    from ground_fusion_b200 import _lib
    from ground_fusion_b200.feature_tracker import FeatureTracker, TrackerGroup
    L = _lib.lib()
    fr = frames(120, 6)
    one = FeatureTracker(640, 480, params8(640), 150, 30, 1, 1)
    for t, g, d in fr[:2]:
        one.trackImageRaw(t, g, d)
    l0 = L.gf_kernel_launch_count()
    one.trackImageRaw(*fr[2])
    per_frame = L.gf_kernel_launch_count() - l0
    one.close()
    for K in (1, 4, 16):
        _, mem = pair(K)
        G = TrackerGroup(mem)
        tk = lambda k: ([fr[k][0]] * K, [fr[k][1].ctypes.data] * K, [fr[k][2].ctypes.data] * K)   # noqa: E731
        for k in range(2):
            G.submit(*tk(k)); G.wait()
        l0 = L.gf_kernel_launch_count()
        G.submit(*tk(2)); G.wait()
        assert L.gf_kernel_launch_count() - l0 == per_frame, K
        mem[K - 1].setPrediction({1: (0.0, 0.0, 2.0)})
        l0 = L.gf_kernel_launch_count()
        G.submit(*tk(3)); G.wait()
        assert L.gf_kernel_launch_count() - l0 == per_frame + 1, K
        G.close()
        close(mem)


def test_equalize_changed_after_create_is_refused():
    """gf_tracker_set_equalize is accepted before a member's first frame, also after the group exists; the group keeps the
    setting the members had at creation and refuses to step members whose setting changed."""
    from ground_fusion_b200._lib import GfError
    from ground_fusion_b200.feature_tracker import TrackerGroup
    S = 2
    ref, mem = pair(S)
    fr = [frames(140 + i, 2) for i in range(S)]
    G = TrackerGroup(mem)
    step = lambda k: ([fr[i][k][0] for i in range(S)], [fr[i][k][1].ctypes.data for i in range(S)], [fr[i][k][2].ctypes.data for i in range(S)])   # noqa: E731
    for tr in mem:
        tr.set_equalize(40.0, (8, 8))
    with pytest.raises(GfError, match="error -1: member 0: equalize setting changed"):
        G.submit(*step(0))
    for tr in mem:
        tr.set_equalize(40.0, (0, 0))
    for k in range(2):
        G.submit(*step(k))
        for i, (o, st, info, _) in enumerate(G.wait()):
            assert o.tobytes() == ref[i].trackImageRaw(*fr[i][k]).tobytes() and info == ref[i].last_info
    G.close()
    close(ref, mem)


def test_errors_leave_members_usable():
    from ground_fusion_b200 import _lib
    from ground_fusion_b200._lib import GfError
    from ground_fusion_b200.feature_tracker import FeatureTracker, TrackerGroup
    L = _lib.lib()
    S = 3
    ref, mem = pair(S)
    fr = [frames(130 + i, 4) for i in range(S)]
    mk = lambda w, h, mc, **k: FeatureTracker(w, h, params8(w), mc, 30, 1, 1, **k)   # noqa: E731
    others = [mk(650, 490, 150), mk(640, 480, 160), mk(640, 480, 150, equalize=True)]
    for o, what in zip(others, ("image size", "max_cnt", "equalize")):
        with pytest.raises(GfError, match="error -1: member 3: %s" % what):
            TrackerGroup(mem + [o])
    close(others)
    with pytest.raises(GfError, match="error -1: member 2: the same tracker listed twice"):
        TrackerGroup([mem[0], mem[1], mem[0]])
    t, g, d = fr[1][0]
    mem[1].submit(t, g, d)
    with pytest.raises(GfError, match="error -1: member 1: has a frame in flight"):
        TrackerGroup(mem)
    mem[1].wait()
    ref[1].trackImageRaw(t, g, d)
    mem[2].set_profiling(True)
    with pytest.raises(GfError, match="error -1: member 2: is in profiling mode"):
        TrackerGroup(mem)
    mem[2].set_profiling(False)
    h = ctypes.c_void_p()
    for n, code in ((0, -1), (65, -4)):
        arr = (ctypes.c_void_p * max(n, 1))(*([mem[0]._h] * max(n, 1)))
        assert L.gf_tracker_group_create(ctypes.byref(h), arr, n) == code and not h.value
    G = TrackerGroup(mem)
    step = lambda k: ([fr[i][k][0] for i in range(S)], [fr[i][k][1].ctypes.data for i in range(S)], [fr[i][k][2].ctypes.data for i in range(S)])   # noqa: E731
    import torch
    d_gray = torch.from_numpy(fr[1][2][1]).cuda()
    d_depth = torch.from_numpy(fr[1][2][2].view(np.int16)).cuda()
    torch.cuda.synchronize()
    G.submit(*step(1))
    with pytest.raises(GfError, match="frame"):
        mem[0].trackImageRaw(*fr[0][2])
    with pytest.raises(GfError, match="error -1: a group step is in flight"):
        mem[1].submit(*fr[1][2])
    with pytest.raises(GfError, match="error -1: a group step is in flight"):
        mem[1].submitDevice(fr[1][2][0], d_gray.data_ptr(), d_depth.data_ptr())
    with pytest.raises(GfError, match="error -1: previous frame not collected"):
        mem[2].trackBatch([fr[2][2][0]], [fr[2][2][1].ctypes.data], [fr[2][2][2].ctypes.data], boxes=[np.zeros((1, 4), np.int64)])
    with pytest.raises(GfError, match="group step"):
        mem[0].wait()
    with pytest.raises(GfError, match="frame in flight"):
        mem[2].setPrediction({1: (0.0, 0.0, 1.0)})
    G.wait()
    for i in range(S):
        ref[i].trackImageRaw(*fr[i][1])
    bx = [np.zeros((0, 4), np.int64), np.zeros((2, 4), np.int64), np.zeros((101, 4), np.int64)]
    with pytest.raises(GfError, match="error -4: member 2: "):
        G.submit(*step(2), boxes=bx)
    G.submit(*step(2))
    for i, (o, st, info, ib) in enumerate(G.wait()):
        assert o.tobytes() == ref[i].trackImageRaw(*fr[i][2]).tobytes() and np.array_equal(st, ref[i].last_status) and info == ref[i].last_info
    G.close()
    for i in range(S):                     # after the group is gone the members track on their own
        assert mem[i].trackImageRaw(*fr[i][3]).tobytes() == ref[i].trackImageRaw(*fr[i][3]).tobytes()
    close(ref, mem)
