"""A due pump that opens, restarts and closes groups between ticks: the stream of tests/test_group_edit_gpu.py and
tools/bench_group_edits.py.

The shard is tests/timers_model.Peers' 64 K x 3 node.  Every `every` ticks, `k_edits` records are issued before the tick's
step: closes, restarts with multi-run logs (terms and ballots from the group's state at that moment) and fresh opens of closed
gids.  Half of the gids come from the groups listed in the steps around the edit.  Both ends keep the pump contract of
rafting_group_edit_begin: a reply to an RPC planned before an edit of its gid never reaches a later step (`drop_replies`).

`Stream` runs the dense reference: whole-shard steps with the synchronous group calls (and, optionally, the oracle
in lock-step).  `DuePump` replays that stream on compact due steps with d steps in flight, issuing the same edits either with
rafting_group_edit_begin ("edit") or by draining and making the synchronous calls ("sync")."""
from __future__ import annotations

from collections import deque

import numpy as np

from rafting_b200 import abi, compact, engine, workload
from tests import compact_active_model as active
from tests import harness
from tests import timers_model as tm

G, R, ROWS = 65536, 3, 3
F = R - 1


def make_cfg(G_: int = G) -> abi.Cfg:
    return abi.make_cfg(replicas=R, max_groups=G_, max_rows=ROWS, entry_pool_cap=64, heartbeat_ms=100, election_ms=300)


def init_all(G_: int = G) -> np.ndarray:
    init = harness.init_array(G_, terms=1 + np.arange(G_) % 5)
    init["now_ms"] = workload.T0_MS
    return init


def plan_edits(k: int, n: int, near: np.ndarray, closed: set, export, now: int) -> np.ndarray:
    """n edit records (gids increasing) for the boundary before tick k.  export(gids) -> states just before the edit."""
    rng = np.random.default_rng(1000 + k)
    pick = np.concatenate([rng.choice(near, min(len(near), n // 2), replace=False) if len(near) else np.zeros(0, np.int64),
                           rng.choice(G, n, replace=False)])
    u = np.unique(pick)
    gids = np.sort(rng.choice(u, min(n, len(u)), replace=False))
    states = export(gids)
    recs = []
    for g, st in zip(gids.tolist(), states):
        if g in closed:                                            # a fresh open of a closed gid
            recs.append(engine.edit_open(g, term=1 + g % 5, now_ms=now, rand_ms=0 if g % 3 else 40))
        elif rng.random() < 0.5:
            recs.append(engine.edit_close(g))
        else:                                                      # a restart over a stored log of 1..8 term runs
            nr = 1 + g % abi.TERM_RUNS
            last = 4 * nr + int(rng.integers(0, 5))
            runs = [(1 + 4 * j, j + 1) for j in range(nr)]
            term = max(int(st.current_term), nr)
            ballot = int(st.voted_for) if g % 2 else int(rng.integers(-1, R))
            recs.append(engine.edit_open(g, runs=runs if nr > 1 else None, term=term, ballot=ballot, first_index=1, last_index=last,
                                         last_term=nr, commit_index=0, now_ms=now, rand_ms=0 if g % 2 else 25 + g % 50))
    return np.array(recs, dtype=abi.GROUP_EDIT)


def apply_sync(s, recs: np.ndarray):
    """the records through the synchronous calls (an Engine after a drain, or the oracle); a restart is a close and an open,
    since the oracle opens only closed gids"""
    for r in recs:
        g = int(r["gid"])
        s.close_group(g)
        if r["kind"] == abi.EDIT_CLOSE:
            continue
        kw = {k: int(r["init"][k]) for k in abi.GROUP_INIT_DTYPE.names if k != "_pad"}
        s.open_group(g, **kw)
        if r["n_runs"]:
            s.load_runs(g, [(int(x), int(y)) for x, y in r["runs"][:r["n_runs"]].tolist()])


def drop_replies(ib: abi.Inbox, k: int, edited_at: np.ndarray, delay: int):
    """the pump contract: replies at tick k answer plans of tick k - delay; those of gids edited after that plan are dropped"""
    m = (edited_at > k - delay) & (edited_at <= k)
    if m.any():
        ib.ev_meta[:, m] = 0
        ib.ev_tn[:, m] = (0, 0)
        ib.ev_el[:, m] = (0, 0)


class Stream:
    """The reference run, one tick per advance(): the edits before the tick (applied through the synchronous calls), the inbox
    (replies of edited gids dropped) and the dense outbox.  After advance(k) the reference engine holds the state after tick k."""

    def __init__(self, k_edits: int, every: int = 10, first: int = 5, oracle=None):
        self.P = tm.Peers(G, rows=ROWS, lost_at=150, t0=workload.T0_MS)
        self.k_edits, self.every, self.first, self.oracle = k_edits, every, first, oracle
        self.ref = engine.Engine(make_cfg())
        init = init_all()
        self.ref.open_bulk(0, init)
        if oracle is not None:
            oracle.open_bulk(0, init)
        self.inboxes, self.wants, self.edits = [], [], {}
        self.edited_at = np.full(G, -10**9, np.int64)
        self.closed, self.terms, self.prev_ev = set(), init["term"].astype(np.int64), np.zeros(0, np.int64)

    def advance(self, k: int):
        assert k == len(self.inboxes)
        if k >= self.first and (k - self.first) % self.every == 0:
            g = np.arange(G)
            near = np.union1d(self.prev_ev, np.flatnonzero((g % 4 == 3) & (g % 5 == k % 5)))   # listed before / after the edit
            st = self.ref.export_bulk(0, G)
            recs = plan_edits(k, self.k_edits, near, self.closed, lambda gs: [st[int(x)] for x in gs], self.P.now(k - 1))
            apply_sync(self.ref, recs)
            if self.oracle is not None:
                apply_sync(self.oracle, recs)
            for r in recs:
                (self.closed.add if r["kind"] == abi.EDIT_CLOSE else self.closed.discard)(int(r["gid"]))
            self.edited_at[recs["gid"].astype(np.int64)] = k
            self.edits[k] = recs
        ib = self.P.inbox(k, self.wants[k - self.P.DELAY] if k >= self.P.DELAY else None, self.terms)
        drop_replies(ib, k, self.edited_at, self.P.DELAY)
        want = self.ref.step(ib)
        if self.oracle is not None:
            assert want.equal(self.oracle.step(ib, threads=8)) == [], f"reference vs oracle, tick {k}"
        self.inboxes.append(ib)
        self.wants.append(want)
        self.terms = want.current_term.copy()
        self.prev_ev = tm.event_gids(ib)


class DuePump:
    """Compact due steps over each tick's event gids, d steps in flight, the stream's edits issued in `mode` "edit" (enqueued
    with rafting_group_edit_begin) or "sync" (drain every slot, then the synchronous calls).  on_wait(j, cout) sees every
    waited outbox; on_tick(k) runs after step k has been begun.  With a timer, ticks_s gets each tick's time (edit, waits,
    encoding, begin) and edit_s the time of each edit (the call, or the drain and the synchronous calls)."""

    def __init__(self, stream: Stream, d: int, mode: str, cap0: int = 8192):
        self.S, self.d, self.mode, self.cap0 = stream, d, mode, cap0
        self.e = engine.Engine(make_cfg())
        self.e.open_bulk(0, init_all())
        self.steps, self.pending, self.counts = {}, deque(), []
        self.ticks_s, self.edit_s = [], []              # per tick, and per edit tick: host time of the edit (or drain + calls)

    def finish(self, j: int, on_wait):
        tail = self.e.step_wait_compact_due(j % 4)
        ci, cout, host = self.steps[j]
        cout.gids = np.concatenate([host, tail])
        self.counts.append(int(cout.counts[3]))
        if on_wait:
            on_wait(j, cout)
        self.steps[j] = (None, cout, host)

    def run(self, ticks: int, on_wait=None, on_tick=None, timer=None):
        e, d, P = self.e, self.d, self.S.P
        for k in range(ticks):
            if k >= len(self.S.inboxes):
                self.S.advance(k)
            t0 = timer() if timer else 0
            if k in self.S.edits:
                if self.mode == "edit":
                    e.group_edit_begin(self.S.edits[k])
                else:
                    while self.pending:
                        self.finish(self.pending.popleft(), on_wait)
                    apply_sync(e, self.S.edits[k])
                if timer:
                    self.edit_s.append(timer() - t0)
            while len(self.pending) > d:
                self.finish(self.pending.popleft(), on_wait)
            ib = self.S.inboxes[k]
            host = tm.event_gids(ib).astype(np.uint32)
            cap = min(max(self.cap0, 2 * max(self.counts, default=0)), G - len(host))
            ai = compact.due_inbox(tm.slice_inbox(ib, host), cap)
            n = len(host) + cap
            tags = np.full((ROWS, n, F), abi.CTAG_NONE, np.uint8)
            sent_term, sent_inc = np.zeros(n, np.int64), np.zeros(n, np.uint32)
            j = k - P.DELAY
            if j in self.steps and self.steps[j][0] is None:          # the step whose plans these replies answer (waited)
                _, cj, _ = self.steps[j]
                p = active.positions(cj.gids, host, G)
                has, q = p >= 0, np.maximum(p, 0)
                tp = cj.tags(rpc_only=True)
                nh = len(host)
                for r in range(2):
                    tags[r + 1][:nh][has] = tp[r][q[has]]
                sent_term[:nh][has], sent_inc[:nh][has] = cj.current_term[q[has]], cj.incarnation[q[has]]
            ci = compact.encode_inbox(ai, tags, sent_term, sent_inc, sweep=True)
            cout = compact.CompactOutbox(ROWS, n, F, esc_cap=ROWS * n * F + 2 * ROWS * n)
            e.step_begin_compact_due(k % 4, host, cap, ci.sweep, ci.as_c(), None if ci.reqs is None else ci.reqs.as_c(), cout.as_c())
            self.steps[k] = (ci, cout, host)
            self.pending.append(k)
            self.steps.pop(k - P.DELAY - 1, None)
            if timer:
                self.ticks_s.append(timer() - t0)
            if on_tick:
                on_tick(k)
        while self.pending:
            self.finish(self.pending.popleft(), on_wait)
