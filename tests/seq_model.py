"""Sequence windows of the fuzz matrix: a case's stream (tests/harness.py, run_fuzz_case's Fuzzer) recorded closed-loop on the
oracle, cut into windows of at most WINDOW launches, and each window replayed into a SUT with ONE call, the way a pump hands
rafting_step_device_seq a queue of decoded batches.  Inside such a call launch k > 0 follows launch k-1 directly on the step
stream, and when it runs in pair_kernel it is launched programmatically (tests/launch_model.py, `sequence`): its blocks stage
their first inbox rows while the launch ahead of it is still running.  A per-launch driver (run_fuzz_case, which synchronises
between launches) never reaches that overlap.

Every launch steps into its own outbox, poisoned (harness.POISON), and must equal the oracle's; the states of a spread of
groups must equal the oracle's at every window boundary, and those of every group at the end."""
from __future__ import annotations

from dataclasses import dataclass, field

import numpy as np

from rafting_b200 import abi, workload
from tests import harness, launch_model

WINDOW = 12


@dataclass
class Recording:
    """A case's stream as the oracle ran it: the election (stepped singly), the fuzz inboxes and the oracle's outboxes, the
    window cuts, the state of `spread` at the end of every window and of every group at the end.  launches: the launch model
    of every fuzz step inside its window; classes[k]: classify_kernel's class of every position of step k before it ran,
    for the programmatic pair_kernel launches behind another pair_kernel launch."""
    case: harness.FuzzCase
    election: list = field(default_factory=list)
    inboxes: list = field(default_factory=list)
    outs: list = field(default_factory=list)
    windows: list = field(default_factory=list)          # (first, end) fuzz step of each window
    spread: np.ndarray | None = None
    states: dict = field(default_factory=dict)           # end of a window -> {gid: state bytes}
    final: list = field(default_factory=list)            # state bytes of every group at the end
    launches: list = field(default_factory=list)         # launch_model.SeqLaunch per fuzz step
    classes: dict = field(default_factory=dict)

    @property
    def fix(self) -> bool:
        return self.case.cfg().flags != 0


def cuts(steps: int, size: int = WINDOW) -> list[tuple[int, int]]:
    return [(lo, min(lo + size, steps)) for lo in range(0, steps, size)]


def record(case: harness.FuzzCase, steps: int | None = None, size: int = WINDOW, classes: bool = False) -> Recording:
    """Runs `case` closed-loop on the oracle (the stream run_fuzz_case drives) and keeps what a replay compares against."""
    cfg, F, G = case.cfg(), case.R - 1, case.G
    steps = case.steps if steps is None else steps
    ref = harness.OracleSUT(cfg)
    ref.open_bulk(0, case.init())
    rec = Recording(case, windows=cuts(steps, size))
    out = None
    if case.leader_share:
        w1 = workload.make_wl(case.seed, 1, G, F, local_slot=case.local_slot)
        for ph in ((0, 1, 2) if cfg.pre_vote else (0, 2)):
            ib = workload.election_inbox_host(w1, ph, out)
            out = ref.step(ib)
            rec.election.append((ib, out))
    gids = case.gids()
    fz = harness.Fuzzer(cfg, ref, seed=case.seed, rows=case.rows, gids=gids, leader_share=case.leader_share,
                        sweep_every=case.sweep_every, stray_requests=case.stray, t0=harness.T33 if case.wide else 0)
    spread = np.arange(0, G, max(1, G // 97))
    if gids is not None:
        spread = np.union1d(spread, gids[gids < G][:64])
    rec.spread = spread
    for lo, hi in rec.windows:
        for k in range(lo, hi):
            ib = fz.make(out)
            if case.compact:
                ib.flags |= abi.INBOX_COMPACT_GROUPS
            sl = launch_model.sequence(case.R, rec.inboxes[k - 1:k] + [ib] if k > lo else [ib], fix=rec.fix)[-1]
            rec.launches.append(sl)
            if classes and sl.programmatic and sl.predecessor == "pair_kernel":
                rec.classes[k] = launch_model.classes(ref, ib)
            out = ref.step(ib)
            rec.inboxes.append(ib)
            rec.outs.append(out)
        rec.states[hi] = {int(g): harness.state_bytes(ref.export(int(g)), F) for g in spread}
    rec.final = [harness.state_bytes(s, F) for s in ref.export_all()]
    return rec


def _assert_states(rec: Recording, sut, want: dict, where: str):
    F = rec.case.R - 1
    for g, sb in want.items():
        got = sut.export(g)
        if harness.state_bytes(got, F) != sb:
            raise AssertionError(f"group {g} state differs {where}: {got.as_dict()}")


def replay(rec: Recording, sut_factory, restore_window: int | None = None) -> int:
    """Replays `rec` into a fresh SUT: the election launch by launch, then every window with one sut.step_seq call.  With
    restore_window = w, the SUT checkpoints at window w's start, runs it, restores without a host synchronisation
    (sut.restore_async) and runs it again into fresh outboxes: both passes must equal the oracle.  Returns the number of
    windows run."""
    case = rec.case
    sut = sut_factory(case.cfg())
    sut.open_bulk(0, case.init())
    for j, (ib, want) in enumerate(rec.election):
        harness.assert_outbox_equal(want, sut.step(ib), where=f"{case.id}: election step {j}")
    runs = 0
    for w, (lo, hi) in enumerate(rec.windows):
        passes = 1
        if w == restore_window:
            sut.checkpoint()
            passes = 2
        for p in range(passes):
            if p:
                sut.restore_async()
            got = sut.step_seq(rec.inboxes[lo:hi])
            assert len(got) == hi - lo
            for k in range(lo, hi):
                harness.assert_outbox_equal(rec.outs[k], got[k - lo],
                                            where=f"{case.id}: window {w} pass {p}, launch {k - lo} (fuzz step {k})")
            runs += 1
        _assert_states(rec, sut, rec.states[hi], where=f"{case.id}: end of window {w}")
    F = case.R - 1
    for g, sb in enumerate(rec.final):
        if harness.state_bytes(sut.export(g), F) != sb:
            raise AssertionError(f"group {g} state differs {case.id}: end of the stream: {sut.export(g).as_dict()}")
    return runs


class SeqOracleSUT(harness.OracleSUT):
    """The oracle as a sequence SUT: a window is its launches stepped one by one (the CPU rehearsal)."""

    def step_seq(self, inboxes):
        return [self.step(ib) for ib in inboxes]


class SeqEngineSUT(harness.EngineSUT):
    """The engine stepping a window through ONE rafting_step_device_seq call: device-resident inboxes, one poisoned device
    outbox per launch."""

    def step_seq(self, inboxes):
        import torch
        from rafting_b200 import devbatch
        n = len(inboxes)
        dins = [devbatch.DevInbox.from_host(ib, self.dev) for ib in inboxes]
        douts = [devbatch.DevOutbox(ib.rows, ib.n, self.F, harness.gcols(ib, self.G), self.dev, fill=self.fill)
                 for ib in inboxes]
        ics = (abi.InboxC * n)(*[d.as_c() for d in dins])
        ocs = (abi.OutboxC * n)(*[d.as_c() for d in douts])
        torch.cuda.synchronize()
        self.e.step_device_seq(ics, ocs, n)
        torch.cuda.synchronize()
        return [d.to_host() for d in douts]

    def checkpoint(self):
        self.e.checkpoint()

    def restore_async(self):
        self.e.restore(sync=False)
