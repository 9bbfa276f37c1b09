"""Device step sequences against the oracle on the whole fuzz matrix (`-m gpu`): every case's stream, recorded closed-loop on
the oracle, replayed window by window with one rafting_step_device_seq call per window (tests/seq_model.py), every launch
into its own poisoned outbox.  Inside a window the R = 3 cases' pair_kernel launches run programmatically behind the launch
ahead of them: behind pair_kernel, behind a class-sorted launch, behind the FIX step kernel (flagged cases).  Also: a window
replayed after restore(sync=False); gathering sequences (gather=True) into per-launch and into two rotated outboxes; and the
refusals of a call that cannot run, which must leave the stream, the tables and the outboxes untouched."""
import numpy as np
import pytest

from rafting_b200 import abi
from tests import harness, seq_model
from tests.test_cfg_fixes_cpu import FUZZ_IDS, flagged

pytestmark = pytest.mark.gpu

CASES = harness.FUZZ_UNSORTED + harness.FUZZ_SORTED
_BY_ID = {c.id: c for c in CASES}
FLAGGED = [flagged(i) for i in FUZZ_IDS]
# a window replayed after a restore without host synchronisation: unsorted R = 3, an active list with a tail of ids >= G,
# class-sorted R = 3 with stray NO_REQUESTS launches, R = 9 class-sorted
RESTORE_IDS = ["R3-G777", "R3-active1500-compact", "R3-n2048", "R9-n2048"]
# whole-shard cases for the gathering sequences: R = 3 unsorted (pair_kernel), R = 5 class-sorted
GATHER_IDS = ["R3-G777", "5-12"]


@pytest.mark.parametrize("case", [pytest.param(c, id=c.id) for c in CASES] +
                         [pytest.param(c, id=f"{c.id}-flagged") for c in FLAGGED])
def test_windows_on_the_engine(case):
    rec = seq_model.record(case)
    assert seq_model.replay(rec, seq_model.SeqEngineSUT) == len(rec.windows)


@pytest.mark.parametrize("case_id", RESTORE_IDS)
def test_window_replayed_after_an_asynchronous_restore(case_id):
    """The bench's bit-exact replay (checkpoint, run, restore(sync=False), run again) on streams with elections, sweeps and
    active lists: both passes of window 1 equal the oracle, and the stream goes on from there."""
    rec = seq_model.record(_BY_ID[case_id])
    assert len(rec.windows) > 1
    assert seq_model.replay(rec, seq_model.SeqEngineSUT, restore_window=1) == len(rec.windows) + 1


class GatherSUT(seq_model.SeqEngineSUT):
    """Gathering sequences on a world-1 communicator.  rotate=False: every launch into its own poisoned outbox, one call per
    window.  rotate=True: two outboxes, A and B, taken in turn as the bench does at world > 1; each call runs two launches
    (A, B), so that both are read back before the next call writes them again, and the engine must keep A alive until the
    gather of the call before has read it.  After every call the last gathered vector equals the last launch's commit
    column."""

    def __init__(self, cfg, rotate: bool):
        super().__init__(cfg)
        self.e.comm_init(0, 1, None)
        self.rotate, self.pair, self.calls = rotate, None, 0

    def _run(self, inboxes, douts):
        import torch
        from rafting_b200 import devbatch
        n = len(inboxes)
        dins = [devbatch.DevInbox.from_host(ib, self.dev) for ib in inboxes]
        ics = (abi.InboxC * n)(*[d.as_c() for d in dins])
        ocs = (abi.OutboxC * n)(*[d.as_c() for d in douts])
        torch.cuda.synchronize()
        self.e.step_device_seq(ics, ocs, n, gather=True)
        torch.cuda.synchronize()
        got = [d.to_host() for d in douts]
        assert np.array_equal(self.e.allgather_last(), got[-1].commit_index), "the last gather is not the last launch's commits"
        self.calls += 1
        return got

    def step_seq(self, inboxes):
        from rafting_b200 import devbatch
        if not self.rotate:
            return self._run(inboxes, [devbatch.DevOutbox(ib.rows, ib.n, self.F, self.G, self.dev, fill=self.fill)
                                       for ib in inboxes])
        if self.pair is None:
            ib = inboxes[0]
            self.pair = [devbatch.DevOutbox(ib.rows, ib.n, self.F, self.G, self.dev, fill=self.fill) for _ in range(2)]
        got = []
        for j in range(0, len(inboxes), 2):
            part = inboxes[j:j + 2]
            for d in self.pair:
                for t in d.t.values():
                    t.fill_(self.fill)
            got += self._run(part, self.pair[:len(part)])
        return got


@pytest.mark.parametrize("rotate", [False, True], ids=["own-outboxes", "two-rotated"])
@pytest.mark.parametrize("case_id", GATHER_IDS)
def test_gathering_windows(case_id, rotate):
    rec = seq_model.record(_BY_ID[case_id])
    assert rec.case.n_active == 0
    suts = []

    def make(cfg):
        suts.append(GatherSUT(cfg, rotate))
        return suts[-1]
    seq_model.replay(rec, make)
    assert suts[0].calls == (sum((hi - lo + 1) // 2 for lo, hi in rec.windows) if rotate else len(rec.windows))


def _two_launch_call(G=777, later=None):
    """An engine at R = 3 over G groups after the first fuzz step of R3-G777, and two device launches of the stream's next
    steps, each with its own poisoned outbox; `later` replaces the second launch's inbox."""
    import torch
    from rafting_b200 import devbatch
    case = _BY_ID["R3-G777"]
    rec = seq_model.record(case, steps=3)
    sut = seq_model.SeqEngineSUT(case.cfg())
    sut.open_bulk(0, case.init())
    harness.assert_outbox_equal(rec.outs[0], sut.step(rec.inboxes[0]), where="first step")
    ibs = [rec.inboxes[1], later or rec.inboxes[2]]
    dins = [devbatch.DevInbox.from_host(ib, sut.dev) for ib in ibs]
    douts = [devbatch.DevOutbox(ib.rows, ib.n, 2, harness.gcols(ib, G), sut.dev, fill=harness.POISON) for ib in ibs]
    torch.cuda.synchronize()
    return sut, dins, douts, (abi.InboxC * 2)(*[d.as_c() for d in dins]), (abi.OutboxC * 2)(*[d.as_c() for d in douts])


def _assert_refused_untouched(sut, douts, call):
    import torch
    from rafting_b200 import engine
    G = sut.G
    digest, launches = sut.e.digest(0, G), sut.e.counters()[0]
    with pytest.raises(engine.RaftingError):
        call()
    torch.cuda.synchronize()
    assert sut.e.counters()[0] == launches, "a launch was enqueued"
    assert np.array_equal(sut.e.digest(0, G), digest), "the tables changed"
    for d in douts:
        for name, t in d.t.items():
            assert bool((t == harness.POISON).all()), f"outbox column {name} was written"


def test_gathering_sequence_refuses_an_active_launch_before_enqueuing_any():
    """A gather copies max_groups entries of a launch's commit column; a launch on an active list writes only its listed
    groups there (n_active entries under COMPACT_GROUPS).  Such a launch anywhere in a gathering call refuses the whole call."""
    for compact_groups in (False, True):
        later = abi.Inbox(3, 100, 2, gids=np.arange(0, 200, 2))
        later.flags |= abi.INBOX_NO_REQUESTS | (abi.INBOX_COMPACT_GROUPS if compact_groups else 0)
        sut, dins, douts, ics, ocs = _two_launch_call(later=later)
        sut.e.comm_init(0, 1, None)
        _assert_refused_untouched(sut, douts, lambda: sut.e.step_device_seq(ics, ocs, 2, gather=True))


def test_sequence_refusals_enqueue_nothing():
    """A gathering call without a communicator, and a call whose second launch lists more groups than the engine has: the
    first launch is not enqueued either."""
    sut, dins, douts, ics, ocs = _two_launch_call()
    _assert_refused_untouched(sut, douts, lambda: sut.e.step_device_seq(ics, ocs, 2, gather=True))
    ics[1].n_active = sut.G + 1
    ics[1].gids = ics[0].op_meta               # never read: the count is refused first
    _assert_refused_untouched(sut, douts, lambda: sut.e.step_device_seq(ics, ocs, 2))
    # the same launches, accepted once the communicator exists, still equal the oracle
    rec = seq_model.record(_BY_ID["R3-G777"], steps=3)
    sut2, dins2, douts2, ics2, ocs2 = _two_launch_call()
    sut2.e.comm_init(0, 1, None)
    sut2.e.step_device_seq(ics2, ocs2, 2, gather=True)
    import torch
    torch.cuda.synchronize()
    for k in range(2):
        harness.assert_outbox_equal(rec.outs[k + 1], douts2[k].to_host(), where=f"launch {k}")
