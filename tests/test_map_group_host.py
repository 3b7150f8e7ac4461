"""Host logic of the map groups, without a GPU: member-list validation, and replay_group's keyframe and slot bookkeeping with
duck-typed map groups."""
import numpy as np
import pytest

from ground_fusion_b200.dense_map import _members
from ground_fusion_b200.replay import WINDOW_SIZE, add_group_keyframes, keyframe_members, replay_group, slide_slots


def test_member_lists_are_checked_before_the_library():
    assert _members([3, 0, 2], 4).tolist() == [3, 0, 2]
    for bad, msg in (([], "no member"), ([0, 4], "out of range"), ([-1], "out of range"), ([1, 2, 1], "twice")):
        with pytest.raises(ValueError, match=msg):
            _members(bad, 4)


def test_replay_group_grid_maps_require_dense_maps():
    with pytest.raises(ValueError, match="grid_maps requires dense_maps"):
        replay_group([None], [None], [None], [None], 1, grid_maps=[object()])
    with pytest.raises(ValueError, match="one dense map and one grid map per stream"):
        replay_group([None, None], [None] * 2, [None] * 2, [None] * 2, 1, dense_maps=[object()])


def test_slide_slots_follows_slidewindow():
    s = list(range(WINDOW_SIZE + 1))
    slide_slots(s, True)
    assert s == list(range(1, WINDOW_SIZE + 1)) + [WINDOW_SIZE]
    s = list(range(WINDOW_SIZE + 1))
    slide_slots(s, False)
    assert s[WINDOW_SIZE - 1] == WINDOW_SIZE and s[:WINDOW_SIZE - 1] == list(range(WINDOW_SIZE - 1))


class _Est:
    def __init__(self, margin_old, P):
        self.margin_old = margin_old
        self.Ps = np.zeros((WINDOW_SIZE + 1, 3)); self.Ps[WINDOW_SIZE - 2] = P
        self.Rs = np.tile(np.eye(3), (WINDOW_SIZE + 1, 1, 1)); self.Rs[WINDOW_SIZE - 2] *= P[0] + 1


class _Stream:
    def __init__(self, i):
        self.i = i

    def color(self, j):
        return np.full((2, 2, 3), 10 * self.i + j, np.uint8)

    def frame(self, j):
        return j, None, np.full((2, 2), 100 * self.i + j, np.uint16)


class _DenseGroup:
    def __init__(self, fail=()):
        self.calls, self.fail = [], fail

    def addKeyFrames(self, members, Rs, Ps, rgbs, depths):
        self.calls.append((list(members), [np.array(R) for R in Rs], [np.array(P) for P in Ps], rgbs, depths))
        return np.ones(len(members), np.int32), np.array([-4 if i in self.fail else 0 for i in members], np.int32)


class _GridGroup:
    def __init__(self):
        self.calls = []

    def addDenseKeyFrames(self, dg, members, Rs, Ps):
        self.calls.append((dg, list(members), [np.array(P) for P in Ps]))
        return np.zeros(len(members), np.int32)


def test_group_keyframes_follow_replays_rule():
    """MARGIN_OLD members whose window frame WINDOW_SIZE - 2 moved add one keyframe each, with the colour and depth of the stream
    frame in that slot; a repeated position is skipped; the grid group gets the same members and poses."""
    ests = [_Est(True, [1.0, 0, 0]), _Est(False, [2.0, 0, 0]), _Est(True, [3.0, 0, 0])]
    last_P = [None, None, np.array([3.0, 0, 0])]          # stream 2's position repeats its last keyframe's
    assert keyframe_members(ests, last_P) == [0]
    slots = [[10 * i + s for s in range(WINDOW_SIZE + 1)] for i in range(3)]
    dg, gg = _DenseGroup(), _GridGroup()
    assert add_group_keyframes(dg, gg, [_Stream(i) for i in range(3)], ests, slots, last_P) == [0]
    members, Rs, Ps, rgbs, depths = dg.calls[0]
    j = slots[0][WINDOW_SIZE - 2]
    assert members == [0] and np.array_equal(Ps[0], [1.0, 0, 0]) and np.array_equal(Rs[0], 2 * np.eye(3))
    assert rgbs[0][0, 0, 0] == j and depths[0][0, 0] == j
    assert gg.calls == [(dg, [0], gg.calls[0][2])] and np.array_equal(gg.calls[0][2][0], [1.0, 0, 0])
    assert np.array_equal(last_P[0], [1.0, 0, 0])
    ests[1].margin_old = True
    assert add_group_keyframes(dg, None, [_Stream(i) for i in range(3)], ests, slots, last_P) == [1]   # stream 0 repeats now
    assert len(gg.calls) == 1
    ests[0].Ps[WINDOW_SIZE - 2] = [5.0, 0, 0]
    ests[2].Ps[WINDOW_SIZE - 2] = [6.0, 0, 0]
    from ground_fusion_b200._lib import GfError
    with pytest.raises(GfError, match="member status"):
        add_group_keyframes(_DenseGroup(fail=(2,)), gg, [_Stream(i) for i in range(3)], ests, slots, last_P)
