"""CPU-only checks behind the streaming kinds' device submits and wide streams: the emission-group rule of
acarsdec_b200.sharding (the one acb_set_emission_groups applies, context.cu acb::stream_groups) on hand-worked cases for
all three units, and the new entry points in the built library and its ctypes binding."""
import ctypes as C

from acarsdec_b200 import api, sharding
from acarsdec_b200.sharding import GROUP_INPUT, GROUP_OUTPUTS, GROUP_SUBMIT, group_of, stream_groups

DEVICE_CALLS = {"acb_submit_real_device": 4, "acb_submit_cs16_device": 4, "acb_submit_cs16_planar_device": 5}


def test_groups_per_submit():
    assert stream_groups(GROUP_SUBMIT, 0, 160, 500, 300) == [500]
    assert stream_groups(GROUP_SUBMIT, 0, 160, 0, 1) == [0]
    assert stream_groups(GROUP_SUBMIT, 0, 160, 500, 0) == []          # no row, no group


def test_groups_every_period_outputs():
    assert stream_groups(GROUP_OUTPUTS, 1000, 200, 500, 300) == [500]
    assert stream_groups(GROUP_OUTPUTS, 1000, 200, 900, 300) == [900, 1000]
    assert stream_groups(GROUP_OUTPUTS, 1000, 200, 1000, 2001) == [1000, 2000, 3000]
    assert stream_groups(GROUP_OUTPUTS, 1000, 200, 999, 1) == [999]
    assert stream_groups(GROUP_OUTPUTS, 1000, 200, 999, 0) == []


def test_groups_per_input_transfer():
    # K = 200, transfers of 65536 samples: transfer t starts a group at output t*65536 // 200
    assert stream_groups(GROUP_INPUT, 65536, 200, 0, 1000) == [0, 327, 655, 983]
    assert stream_groups(GROUP_INPUT, 65536, 200, 327, 1) == [327]          # transfer 1 began before output 327 did
    assert stream_groups(GROUP_INPUT, 65536, 200, 328, 1000) == [328, 655, 983, 1310]
    # transfers shorter than a row: transfer 0 (samples 0..149) completes no row, transfer 1 completes output 0, which
    # transfer 0 began, so both share the submit's first group
    assert stream_groups(GROUP_INPUT, 150, 200, 0, 3) == [0, 1, 2]
    # four 50-sample transfers per row: only every fourth starts a new group
    assert stream_groups(GROUP_INPUT, 50, 200, 0, 2) == [0, 1]
    assert stream_groups(GROUP_INPUT, 50, 200, 5, 3) == [5, 6, 7]


def test_group_of_and_merge_order():
    starts = [0, 327, 655]
    assert [group_of(starts, p) for p in (0, 326, 327, 654, 655, 10 ** 6)] == [1, 1, 2, 2, 3, 3]
    # (block, stream, chn, pos) tuples of two ranks, each in its own emission order: merged by (group, stream, chn, pos)
    rank0 = [(0, 0, 0, 100), (0, 0, 0, 400), (0, 0, 1, 330)]
    rank1 = [(0, 0, 2, 10), (0, 0, 3, 700), (0, 0, 2, 660)]
    merged = sharding.merge_messages([rank0, rank1], key=lambda m: (group_of(starts, m[3]),) + m[1:4])
    assert [m[2:] for m in merged] == [(0, 100), (2, 10), (0, 400), (1, 330), (2, 660), (3, 700)]


def test_device_calls_are_exported_and_bound(native):
    bound = {name: (res, args) for name, res, args in api.ABI}
    for name, nargs in DEVICE_CALLS.items():
        assert hasattr(native, name)
        res, args = bound[name]
        assert res is C.c_int and len(args) == nargs
        assert getattr(api.Context, name[len("acb_"):])
