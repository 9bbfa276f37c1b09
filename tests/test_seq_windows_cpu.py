"""The sequence windows of tests/test_seq_windows_gpu.py without a GPU: every window of every case replayed with the oracle on
both sides, the launch model of a rafting_step_device_seq call, what the windows reach among its programmatic pair_kernel
launches (the launches that overlap the one ahead of them), and a SUT that hands back the wrong launch's outbox is caught."""
import functools

import numpy as np
import pytest

from rafting_b200 import abi
from tests import harness, launch_model, seq_model
from tests.test_cfg_fixes_cpu import FUZZ_IDS, flagged

CASES = harness.FUZZ_UNSORTED + harness.FUZZ_SORTED
FLAGGED = [flagged(i) for i in FUZZ_IDS]
ALL = [pytest.param(c, id=c.id) for c in CASES] + [pytest.param(c, id=f"{c.id}-flagged") for c in FLAGGED]


@functools.lru_cache(maxsize=None)
def recorded(case) -> seq_model.Recording:
    return seq_model.record(case, classes=True)


def test_sequence_model_examples():
    def ib(n, flags=0):
        x = abi.Inbox(1, n, 2)
        x.flags = flags
        return x
    NR = abi.INBOX_NO_REQUESTS
    s = launch_model.sequence(3, [ib(777), ib(777, NR), ib(2048), ib(2048, NR)])
    assert [x.programmatic for x in s] == [False, True, False, True]
    assert [x.predecessor for x in s] == [None, "pair_kernel", "pair_kernel", "step_kernel<2,3>"]
    assert s[3].after == ("classify_kernel", "slow_kernel<2,4>", "step_kernel<2,3>")
    assert not any(x.programmatic for x in launch_model.sequence(3, [ib(777), ib(777)], gather=True))
    f = launch_model.sequence(3, [ib(777), ib(777, NR), ib(777, NR)], fix=True)
    assert [x.kernels[-1] for x in f] == ["step_kernel<2,3,true>", "pair_kernel", "pair_kernel"]
    assert [x.programmatic for x in f] == [False, True, True]
    assert not any(x.programmatic for x in launch_model.sequence(5, [ib(777), ib(777, NR)]))


@pytest.mark.parametrize("case", ALL)
def test_windows_on_the_oracle(case):
    """Every window of the case, the oracle on both sides: the recording replays, window by window, to the same outboxes and
    states."""
    rec = recorded(case)
    assert seq_model.replay(rec, seq_model.SeqOracleSUT) == len(rec.windows)
    assert all(hi - lo <= seq_model.WINDOW for lo, hi in rec.windows)


def test_windows_reach_every_predecessor_of_a_programmatic_launch():
    """Across the matrix, programmatic pair_kernel launches follow pair_kernel, a class-sorted R = 3 launch (the sorted cases'
    stray NO_REQUESTS launches) and the FIX step kernel (the flagged cases)."""
    after = {}
    for case in CASES + FLAGGED:
        for sl in recorded(case).launches:
            if sl.programmatic:
                after[sl.after] = after.get(sl.after, 0) + 1
    assert after.get(("pair_kernel",), 0) > 0, after
    assert after.get(("classify_kernel", "slow_kernel<2,4>", "step_kernel<2,3>"), 0) > 0, after
    assert after.get(("step_kernel<2,3,true>",), 0) > 0, after


def test_pair_behind_pair_launches_reach_every_class_sweeps_and_tails():
    """Among the programmatic pair_kernel launches behind another pair_kernel launch: positions in all four classes, sweep
    rows, and an active list whose tail holds ids >= max_groups."""
    seen, sweeps, tails, n = np.zeros(launch_model.NCLS, np.int64), 0, 0, 0
    for case in CASES + FLAGGED:
        rec = recorded(case)
        for k, cls in rec.classes.items():
            ib = rec.inboxes[k]
            n += 1
            seen += np.bincount(cls, minlength=launch_model.NCLS)
            sweeps += int(ib.row_now is not None and (ib.row_now != 0).any())
            tails += int(ib.gids is not None and (ib.gids >= case.G).any())
    assert n > 100, n
    assert (seen > 0).all(), seen.tolist()
    assert sweeps > 0 and tails > 0, (sweeps, tails)


class _HandsBackTheLastOutbox(seq_model.SeqOracleSUT):
    """A sequence SUT that, in its second window, returns launch k's outbox for launch k + 1."""
    calls = 0

    def step_seq(self, inboxes):
        outs = super().step_seq(inboxes)
        type(self).calls += 1
        if type(self).calls == 2:
            k = len(outs) // 2
            outs[k + 1] = outs[k]
        return outs


def test_windows_catch_an_outbox_handed_to_the_wrong_launch():
    _HandsBackTheLastOutbox.calls = 0
    with pytest.raises(AssertionError, match="window 1 pass 0, launch 7"):
        seq_model.replay(recorded(harness.FUZZ_UNSORTED[0]), _HandsBackTheLastOutbox)
