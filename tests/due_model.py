"""Due steps on the compact host path (rafting_step_begin_compact_due) — TEST INFRASTRUCTURE: the tail the device chooses,
restated in numpy, and a pump that lists only each step's event gids and lets the tail add the due groups.

  tail      the tail of a due step over the host's list at sweep time `until`: the due groups outside the list, lowest first, up
            to cap, then fillers (groups outside the list that are not due), lowest first, until it holds cap; and the full
            number of due groups outside the list (counts[3])
  DuePump   a system under test that turns every whole-shard step into the due step over the step's own event gids plus the
            model's tail of the state the step sees, on an inner SUT that takes active lists.  Its cap follows the counts[3] of
            the steps it has waited for, d steps behind: the only thing pipelining changes for a due pump"""
from __future__ import annotations

import numpy as np

from rafting_b200 import abi
from tests import timers_model as tm


def tail(t: dict, host: np.ndarray, cap: int, until: int) -> tuple[np.ndarray, int]:
    """-> (the tail, uint32 [cap], and the number of due groups outside host); t: timers_model.table of the state the step sees"""
    G = len(t["timer"])
    listed = np.zeros(G, bool)
    listed[np.asarray(host, np.int64)] = True
    d = tm.due(t, until)
    due_out, idle_out = np.flatnonzero(d & ~listed), np.flatnonzero(~d & ~listed)
    k = min(len(due_out), cap)
    return np.concatenate([due_out[:k], idle_out[:cap - k]]).astype(np.uint32), len(due_out)


class DuePump:
    """Whole-shard steps in, due steps out (event gids + the model's tail) run on `inner`, whole-shard outboxes back.
    listed[k]: groups step k listed; counts[k]: its counts[3]; overflows: steps whose counts[3] exceeded their cap."""

    def __init__(self, inner, G: int, F: int, d: int, cap0: int):
        self.inner, self.G, self.F, self.d, self.cap0 = inner, G, F, d, cap0
        self.cfg = getattr(inner, "cfg", None)
        self.last = None
        self.listed, self.counts, self.fillers, self.overflows = [], [], 0, 0

    def _table(self) -> dict:
        if hasattr(self.inner, "export_bulk"):
            return tm.table(self.inner.export_bulk(0, self.G))
        return tm.table([self.inner.export(g) for g in range(self.G)])

    def open_bulk(self, first, init):
        self.inner.open_bulk(first, init)

    def export(self, g):
        return self.inner.export(g)

    def log_term(self, g, i):
        return self.inner.log_term(g, i)

    def cap(self, n_host: int) -> int:
        """twice the largest counts[3] among the steps waited for (all but the d in flight), at least cap0, at most what fits"""
        seen = self.counts[:max(len(self.counts) - self.d, 0)]
        return min(max(self.cap0, 2 * max(seen, default=0)), self.G - n_host)

    def step(self, ib: abi.Inbox) -> abi.Outbox:
        until = int(ib.row_now.max()) if ib.row_now is not None else 0
        host = tm.event_gids(ib)
        cap = self.cap(len(host))
        if self.last is None or cap == 0:                 # the first step lists every group: its outbox holds every group
            L = np.arange(self.G, dtype=np.uint32)        # column (and when every group has an event, so does the list)
        elif until == 0:                                  # no sweep row: an active step over the events
            L = host.astype(np.uint32)
        else:
            tl, n_due = tail(self._table(), host, cap, until)
            self.counts.append(n_due)
            self.overflows += int(n_due > cap)
            self.fillers += cap - min(n_due, cap)
            L = np.concatenate([host.astype(np.uint32), tl])
        self.listed.append(len(L))
        S = np.sort(L)
        if len(S):
            out = tm.expand_outbox(self.inner.step(tm.slice_inbox(ib, S)), S, self.last, self.G)
        else:
            out = tm.expand_outbox(abi.Outbox(ib.rows, 0, self.F, 0), S, self.last, self.G)
        self.last = out
        return out
