"""Timers on the compact host path — TEST INFRASTRUCTURE: the due predicate over exported state, and the pipelining rule of
include/rafting_b200.h ("PIPELINING RULE") as a pump that lists groups by it.

  due / next_deadline   the sweep's predicate (step_body.inc, pair_kernel.cuh) restated in numpy over (timer, role, alive)
  RulePump              a system under test that turns every whole-shard step it is given into the step over the rule's
                        list: due(state after step k-d, until = the step's last sweep time) u the event gids of the d steps
                        in flight and of the step itself.  It runs that step on an inner SUT that takes active lists (the
                        oracle, or the engine) and hands back the whole-shard outbox the step stands for"""
from __future__ import annotations

import numpy as np

from rafting_b200 import abi

I64MAX = np.iinfo(np.int64).max


def table(states) -> dict:
    """timer, role and alive of exported group states (abi.GroupState sequence)."""
    return dict(timer=np.array([s.timer for s in states], np.int64), role=np.array([s.role for s in states], np.int64),
                alive=np.array([s.alive for s in states], np.int64))


def due(t: dict, until: int) -> np.ndarray:
    """alive && (leader ? timer <= t : timer > 0 && timer != INT64_MAX && timer <= t), as a bool mask over the groups"""
    timer, leader, alive = t["timer"], t["role"] == abi.ROLE_LEADER, t["alive"] != 0
    return alive & np.where(leader, timer <= until, (timer > 0) & (timer != I64MAX) & (timer <= until))


def next_deadline(t: dict, until: int) -> int:
    """the earliest deadline after until that a later sweep would fire, or INT64_MAX"""
    timer, leader, alive = t["timer"], t["role"] == abi.ROLE_LEADER, t["alive"] != 0
    armed = alive & (leader | ((timer > 0) & (timer != I64MAX))) & (timer > until)
    return int(timer[armed].min()) if armed.any() else int(I64MAX)


def event_gids(ib: abi.Inbox) -> np.ndarray:
    """groups with a group op outside the sweep rows, or a lane event, in a whole-shard inbox"""
    has = np.zeros(ib.n, bool)
    sweep = ib.row_now if ib.row_now is not None else np.zeros(ib.rows, np.int64)
    if ib.op_meta is not None:
        has |= ((ib.op_meta[sweep == 0] & np.uint64(0xFF)) != 0).any(axis=0)
    if ib.ev_meta is not None:
        has |= ((ib.ev_meta & np.uint64(0xF)) != 0).any(axis=(0, 2))
    return np.flatnonzero(has)


def slice_inbox(ib: abi.Inbox, gids: np.ndarray) -> abi.Inbox:
    """The whole-shard inbox ib restricted to the active list gids (positional columns, COMPACT_GROUPS)."""
    a = abi.Inbox.__new__(abi.Inbox)
    a.rows, a.n, a.F = ib.rows, len(gids), ib.F
    a.gids = np.ascontiguousarray(gids, dtype=np.uint32)
    a.row_now = ib.row_now
    g = gids.astype(np.int64)
    for name in ("op_meta", "op_nr", "op_ab", "op_cd", "op_e", "ev_meta", "ev_tn", "ev_el"):
        col = getattr(ib, name)
        setattr(a, name, None if col is None else np.ascontiguousarray(col[:, g]))
    a.ent_terms, a.ent_count = ib.ent_terms, ib.ent_count
    a.flags = ib.flags | abi.INBOX_COMPACT_GROUPS
    return a


def expand_outbox(o: abi.Outbox, gids: np.ndarray, last: abi.Outbox | None, G: int) -> abi.Outbox:
    """The whole-shard outbox an active step stands for: row columns zero outside the list, group columns of an unlisted group
    as the last step left them, without the per-step dirty bits (role_word bits 30 / 31)."""
    w = abi.Outbox(o.rows, G, o.F, G)
    g = gids.astype(np.int64)
    for name, _, _ in abi.Outbox.ROW_COLS:
        getattr(w, name)[:, g] = getattr(o, name)
    for name, _ in abi.Outbox.GROUP_COLS:
        if last is not None:
            getattr(w, name)[...] = getattr(last, name)
        getattr(w, name)[g] = getattr(o, name)[:len(g)]
    keep = np.ones(G, bool); keep[g] = False
    w.role_word[keep] &= np.uint32(0x3FFFFFFF)
    return w


class RulePump:
    """Whole-shard steps in, steps over the rule's list run on `inner` (anything with step / export_bulk or export), whole-shard
    outboxes out.  d: steps in flight behind the one being encoded.  listed[k]: how many groups step k listed."""

    def __init__(self, inner, G: int, F: int, d: int):
        self.inner, self.G, self.F, self.d = inner, G, F, d
        self.cfg = getattr(inner, "cfg", None)
        self.hist = None                         # hist[j]: the timer table after j steps (from open_bulk on)
        self.lists: list[np.ndarray] = []
        self.events: list[np.ndarray] = []
        self.last = None
        self.listed, self.due_only = [], 0        # due_only: groups listed by the due query alone (no event, not in flight)

    def _table(self) -> dict:
        if hasattr(self.inner, "export_bulk"):
            return table(self.inner.export_bulk(0, self.G))
        return table([self.inner.export(g) for g in range(self.G)])

    def open_bulk(self, first, init):
        self.inner.open_bulk(first, init)
        self.hist = [self._table()]

    def export(self, g):
        return self.inner.export(g)

    def log_term(self, g, i):
        return self.inner.log_term(g, i)

    def rule(self, ib: abi.Inbox) -> np.ndarray:
        j = len(self.lists)
        if self.hist is None:
            self.hist = [self._table()]
        until = int(ib.row_now.max()) if ib.row_now is not None else 0
        q = np.flatnonzero(due(self.hist[max(j - self.d, 0)], until)) if until else np.zeros(0, np.int64)
        flight = [self.events[k] for k in range(max(j - self.d, 0), j)]
        ev = event_gids(ib)
        self.events.append(ev)
        if self.last is None:                    # the first step lists every group: its outbox holds every group column
            return np.arange(self.G, dtype=np.uint32)
        self.due_only += len(np.setdiff1d(q, np.concatenate([ev] + flight)))
        return np.union1d(np.union1d(q, ev), np.concatenate(flight) if flight else np.zeros(0, np.int64)).astype(np.uint32)

    def step(self, ib: abi.Inbox) -> abi.Outbox:
        L = self.rule(ib)
        self.lists.append(L.astype(np.int64))
        self.listed.append(len(L))
        if len(L):
            out = expand_outbox(self.inner.step(slice_inbox(ib, L)), L, self.last, self.G)
        else:                                    # nothing fires, nothing arrives: the step leaves the shard as it is
            out = expand_outbox(abi.Outbox(ib.rows, 0, self.F, 0), L, self.last, self.G)
        self.last = out
        self.hist.append(self._table())
        return out


class Peers:
    """The two remote nodes of a 3-node shard at local slot 0 (lane f = node slot f + 1), as a deterministic stream of whole-shard
    inboxes of `rows` >= 3 rows, one per 10 ms tick.  Row 0 is the sweep row (row_now[0] = the tick's time) and carries nothing
    else, so every plan or ballot in row 0 of an outbox was fired by a timer.
      * groups g % 4 == 1 and 3 have their leader at slot 1: a heartbeat AppendEntries (row 1) every 50 ms keeps them followers;
        the leader of the g % 4 == 1 groups disappears at tick `lost_at`, and those groups elect
      * groups g % 2 == 0 have no leader from the start: their election timers fire, they elect and then lead
      * every AppendEntries / InstallSnapshot plan and every ballot of rows 0 and 1 is answered 4 ticks later, in the next row
        (success / granted), so that a pump running 4 steps in flight has the planning step's tags when it encodes the reply"""

    DELAY = 4

    def __init__(self, G: int, rows: int = 3, lost_at: int = 150, t0: int = 1_700_000_000_000):
        assert rows >= 3
        self.G, self.F, self.rows, self.lost_at, self.t0 = G, 2, rows, lost_at, t0
        self.g = np.arange(G)
        self.terms = None

    def now(self, k: int) -> int:
        return self.t0 + 10 * (k + 1)

    def inbox(self, k: int, planned: abi.Outbox | None, terms: np.ndarray) -> abi.Inbox:
        """Tick k.  planned: the whole-shard outbox of tick k - DELAY (None before); terms: every group's current term."""
        G, F, rows, now = self.G, self.F, self.rows, self.now(k)
        ib = abi.Inbox(rows, G, F, ent_cap=1, sweep=True)
        ib.row_now[0] = now
        g = self.g
        led = ((g % 4 == 3) | ((g % 4 == 1) & (k < self.lost_at))) & (k % 5 == g % 5)
        at = np.flatnonzero(led)
        ib.op_meta[1, at] = abi.op_make(abi.OP_AE_REQUEST, 1)
        ib.op_nr["x"][1, at] = now
        ib.op_ab["x"][1, at] = terms[at]                                     # term; prevLogIndex 0
        ib.op_e[1, at] = 1
        if planned is not None:
            for r in range(2):
                pm = planned.plan_meta[r]
                kind = (pm & U64(0xF)).astype(np.int64)
                ack = (kind == abi.PLAN_AE) | (kind == abi.PLAN_IS)
                ev = np.where(ack, (np.where(kind == abi.PLAN_IS, abi.EV_IS_ACK, abi.EV_AE_ACK).astype(np.uint64) |
                                    (U64(abi.OUT_OK) << U64(4)) | (U64(1) << U64(6)) | ((pm >> U64(32)) << U64(32))), U64(0))
                ib.ev_meta[r + 1] = ev
                ib.ev_tn["x"][r + 1] = np.where(ack, planned.current_term[:, None], 0)
                ib.ev_tn["y"][r + 1] = np.where(ack, now, 0)
                ib.ev_el["x"][r + 1] = np.where(ack, planned.plan_epoch[r], 0)
                ib.ev_el["y"][r + 1] = np.where(ack, planned.plan_lc["x"][r], 0)
                bm = planned.ballot_meta[r]
                bk = (bm & U64(0xF)).astype(np.int64)
                has = (bk == abi.BALLOT_PREVOTE) | (bk == abi.BALLOT_VOTE)
                rk = np.where(bk == abi.BALLOT_PREVOTE, abi.EV_PV_REPLY, abi.EV_RV_REPLY).astype(np.uint64)
                vote = rk | (U64(abi.OUT_OK) << U64(4)) | (U64(1) << U64(6)) | ((bm >> U64(32)) << U64(32))
                rt = np.where(bk == abi.BALLOT_PREVOTE, planned.ballot_term[r] - 1, planned.ballot_term[r])
                for f in range(F):
                    ib.ev_meta[r + 1, has, f] = vote[has]
                    ib.ev_tn["x"][r + 1, has, f] = rt[has]
                    ib.ev_tn["y"][r + 1, has, f] = now
                    ib.ev_el[r + 1, has, f] = (0, 0)
        return ib


U64 = np.uint64
