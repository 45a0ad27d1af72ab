"""The emission-group rule for streams at different positions (ragged submits, acb_reset_stream), on the CPU.

sharding.group_number numbers a stream's groups from its own start; within a submit frames leave in (group number,
stream, channel, time) order.  Checked here against a model that counts the group starts one by one, for every unit, at
positions that are and are not group starts, and against stream_groups: within one submit the numbers of its starts
are consecutive, and with every stream at the same position the order is stream_groups' (group index, stream, ...)."""
import random

import pytest

from acarsdec_b200 import sharding
from acarsdec_b200.sharding import GROUP_INPUT, GROUP_OUTPUTS, GROUP_SUBMIT

UNITS = [(None, 0), (GROUP_SUBMIT, 0), (GROUP_OUTPUTS, 1), (GROUP_OUTPUTS, 512), (GROUP_OUTPUTS, 1024),
         (GROUP_INPUT, 65536), (GROUP_INPUT, 200 * 1024 + 7), (GROUP_INPUT, 160), (GROUP_INPUT, 100), (GROUP_INPUT, 37)]


def model_number(unit, period, K, pos):
    """Group starts in (0, pos], counted one by one."""
    if unit is None:
        return sum(1 for b in range(1, pos + 1) if b % 1024 == 0)
    if unit == GROUP_SUBMIT:
        return 0
    if unit == GROUP_OUTPUTS:
        return sum(1 for b in range(1, pos + 1) if b % period == 0)
    starts, t = set(), 1
    while t * period // K <= pos:
        starts.add(t * period // K)
        t += 1
    return len(starts - {0})


@pytest.mark.parametrize("unit,period", UNITS)
def test_number_matches_model(unit, period):
    rng = random.Random(7)
    K = 160
    for pos in list(range(0, 40)) + [1023, 1024, 1025, 4095, 4096] + [rng.randrange(0, 20000) for _ in range(40)]:
        assert sharding.group_number(unit, period, K, pos) == model_number(unit, period, K, pos), pos


def _starts(unit, period, K, pos, n):
    if unit is None:
        return [pos + 1024 * b for b in range(n // 1024)]
    return sharding.stream_groups(unit, period, K, pos, n)


@pytest.mark.parametrize("unit,period", [u for u in UNITS if u[0] != GROUP_SUBMIT])
def test_submit_starts_are_consecutive_numbers(unit, period):
    """A submit's first start carries the number of the group it continues; every further start is the next number."""
    rng = random.Random(11)
    K = 200
    for _ in range(60):
        n = 1024 * rng.randrange(1, 5) if unit is None else rng.randrange(1, 5000)
        pos = 1024 * rng.randrange(0, 50) if unit is None else rng.randrange(0, 50000)
        g = _starts(unit, period, K, pos, n)
        nums = [sharding.group_number(unit, period, K, p) for p in g]
        assert nums == list(range(nums[0], nums[0] + len(nums)))
        # every sample of the submit has the number of the last start at or before it
        for p in sorted(rng.sample(range(pos, pos + n), min(n, 20))):
            assert sharding.group_number(unit, period, K, p) == nums[sharding.group_of(g, p) - 1]


def _order(frames, key):
    return [f for _, f in sorted((key(f), f) for f in frames)]


@pytest.mark.parametrize("unit,period", UNITS)
def test_equal_positions_give_the_lockstep_order(unit, period):
    """Streams at one position, counts equal or not (zero included): the per-stream key orders frames as the lockstep
    key (index of the group in the submit's starts, stream, channel, time) does."""
    rng = random.Random(3)
    K = 160
    for _ in range(40):
        pos = 1024 * rng.randrange(0, 30) if unit is None else rng.randrange(0, 30000)
        rows = [(1024 * rng.randrange(0, 4) if unit is None else rng.choice([0, rng.randrange(1, 4000)])) for _ in range(5)]
        if max(rows) == 0:
            continue
        shared = _starts(unit, period, K, pos, max(rows))
        frames = [(s, rng.randrange(8), pos + rng.randrange(r)) for s, r in enumerate(rows) if r for _ in range(6)]
        lockstep = _order(frames, lambda f: (sharding.group_of(shared, f[2]), f[0], f[1], f[2]))
        ragged = _order(frames, lambda f: (sharding.group_number(unit, period, K, f[2]), f[0], f[1], f[2]))
        assert ragged == lockstep


def test_streams_at_different_positions():
    """A stream behind the others (a stall, a reset) emits its earlier groups first within the submit."""
    K = 160
    frames = [(0, 0, 5000), (1, 0, 10), (1, 1, 1100), (2, 3, 5100)]
    key = lambda f: (sharding.group_number(None, 0, K, f[2]), f[0], f[1], f[2])   # noqa: E731
    assert _order(frames, key) == [(1, 0, 10), (1, 1, 1100), (0, 0, 5000), (2, 3, 5100)]
