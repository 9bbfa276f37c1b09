"""Due steps on the compact host path (`-m gpu`): rafting_step_begin_compact_due, whose list is the host's gids followed by a
tail the device chooses right before the step.

  * a 64 K x 3 closed loop of 320 ticks of tests/timers_model.Peers on due steps over each tick's event gids, d = 0 and d = 3
    steps in flight: every waited outbox equals the reference engine's dense whole-shard sweep step at the listed groups, the
    digests equal the reference's and, at the end, the oracle's; heartbeats planned at tail positions are acked at host
    positions; the due lists are smaller than the pipelining rule's lists at d = 3
  * the config #3 storm at R = 5, flags 1 and 5, with caps below and above counts[3]: the tail and counts[3] equal the model
    over rafting_state_export_bulk, and the step equals rafting_step_begin_compact_sweep over the explicit list gids u tail
  * a due query and a due step over an empty host list, in flight in the same slot number on one state: the tail is the
    query's list (cut at cap, or followed by fillers) and counts[3] its n_due
  * refusals leave the slot free; the native runs through the stand-in JNIEnv"""
import ctypes as C
from collections import deque

import numpy as np
import pytest

from oracle import binding
from rafting_b200 import abi, compact, engine, workload
from tests import compact_active_model as active
from tests import compact_model as model
from tests import due_model as dm
from tests import harness
from tests import timers_model as tm
from tests.compact_model import EL, PT

pytestmark = pytest.mark.gpu


def _table_bulk(e, G):
    """timer / role / alive of every group through rafting_state_export_bulk"""
    return tm.table(e.export_bulk(0, G))


def _at(o: abi.Outbox, where: np.ndarray) -> abi.Outbox:
    """the outbox o at the positions `where` (o's group columns by gid when o is a whole-shard outbox of G groups and
    `where` holds gids; by position when o is an active outbox)"""
    p = abi.Outbox(o.rows, len(where), o.F, len(where))
    g = where.astype(np.int64)
    for name, _, _ in abi.Outbox.ROW_COLS:
        getattr(p, name)[...] = getattr(o, name)[:, g]
    for name, _ in abi.Outbox.GROUP_COLS:
        getattr(p, name)[...] = getattr(o, name)[g]
    return p


def _pad(a: np.ndarray | None, cap: int, fill) -> np.ndarray | None:
    """a per-position array of the host's list, extended by cap tail positions of `fill` (axis 1 for [rows, n, ...])"""
    if a is None:
        return None
    axis = 0 if a.ndim == 1 else 1
    shape = list(a.shape); shape[axis] = cap
    return np.concatenate([a, np.full(shape, fill, a.dtype)], axis=axis)


@pytest.mark.parametrize("d", [0, 3])
def test_closed_loop_on_due_steps_matches_whole_shard_sweeps(d):
    """The closed loop of test_closed_loop_on_due_lists_matches_whole_shard_sweeps on due steps: the candidate engine lists only
    each tick's event gids and lets the device add the due groups.  The cap follows the counts[3] of the steps waited for
    (d behind).  Due queries still run on the candidate, only to size the pipelining rule's list for the comparison."""
    import torch
    G, R, rows, ticks = 65536, 3, 3, 320
    F = R - 1
    cfg = abi.make_cfg(replicas=R, max_groups=G, max_rows=rows, entry_pool_cap=64, heartbeat_ms=100, election_ms=300)
    init = harness.init_array(G, terms=1 + np.arange(G) % 5)
    init["now_ms"] = workload.T0_MS
    ref, e, o = engine.Engine(cfg), engine.Engine(cfg), binding.Oracle(cfg)
    for s in (ref, e, o):
        s.open_bulk(0, init)
    P = tm.Peers(G, rows=rows, lost_at=150, t0=workload.T0_MS)
    bufs = [torch.zeros(G, dtype=torch.int32).pin_memory() for _ in range(4)]
    wants, terms, events, steps = [], init["term"].astype(np.int64), {}, {}
    pending = deque()
    listed, rule_listed, counts, tail_acks = [], [], [], 0
    cap0 = 8192

    def begin_query(t):
        e.timers_due_begin(t % 4, P.now(t), bufs[t % 4].data_ptr(), G)

    def finish(j):
        tail = e.step_wait_compact_due(j % 4)
        ci, cout, host = steps[j]
        cout.gids = np.concatenate([host, tail])
        L = cout.gids.astype(np.int64)
        assert len(np.unique(L)) == len(L) and not np.isin(tail, host).any()
        n_due = int(cout.counts[3])
        counts.append(n_due)
        assert n_due <= len(tail), f"step {j}: {n_due} due groups outside the list, cap {len(tail)}"
        harness.assert_outbox_equal(_at(wants[j], cout.gids), compact.decode_outbox(cout), where=f"step {j} (d = {d})")
        steps[j] = (None, cout, host)

    for t in range(d + 1):
        begin_query(t)
    for k in range(ticks):
        ib = P.inbox(k, wants[k - P.DELAY] if k >= P.DELAY else None, terms)
        want = ref.step(ib)
        assert want.equal(o.step(ib, threads=8)) == [], f"reference vs oracle, tick {k}"
        wants.append(want)
        terms = want.current_term.copy()
        while len(pending) > d:
            finish(pending.popleft())
        n_q, _ = e.timers_due_wait(k % 4)
        Q = bufs[k % 4].numpy()[:n_q].view(np.uint32).astype(np.int64)
        events[k] = tm.event_gids(ib)
        flight = [events[j] for j in pending]
        rule_listed.append(len(np.union1d(np.union1d(Q, events[k]), np.concatenate(flight) if flight else np.zeros(0, np.int64))))
        host = events[k].astype(np.uint32)
        cap = min(max(cap0, 2 * max(counts, default=0)), G - len(host))
        listed.append(len(host) + cap)
        ai = compact.due_inbox(tm.slice_inbox(ib, host), cap)
        tags = np.full((rows, len(host), F), abi.CTAG_NONE, np.uint8)
        sent_term, sent_inc = np.zeros(len(host), np.int64), np.zeros(len(host), np.uint32)
        j = k - P.DELAY
        if j in steps and steps[j][0] is None:                           # the step whose plans these acks answer (waited)
            _, cj, hj = steps[j]
            p = active.positions(cj.gids, host, G)
            has, q = p >= 0, np.maximum(p, 0)
            tp = cj.tags(rpc_only=True)
            for r in range(2):
                tags[r + 1][has] = tp[r][q[has]]
            sent_term[has], sent_inc[has] = cj.current_term[q[has]], cj.incarnation[q[has]]
            acked = (ib.ev_meta[1:, host.astype(np.int64)] != 0).any(axis=(0, 2))
            tail_acks += int((acked & has & (p >= len(hj))).sum())        # planned at a tail position, acked at a host one
        ci = compact.encode_inbox(ai, _pad(tags, cap, abi.CTAG_NONE), _pad(sent_term, cap, 0), _pad(sent_inc, cap, 0), sweep=True)
        n = len(host) + cap
        cout = compact.CompactOutbox(rows, n, F, esc_cap=rows * n * F + 2 * rows * n)
        e.step_begin_compact_due(k % 4, host, cap, ci.sweep, ci.as_c(), None if ci.reqs is None else ci.reqs.as_c(), cout.as_c())
        steps[k] = (ci, cout, host)
        pending.append(k)
        steps.pop(k - P.DELAY - 1, None)
        begin_query(k + d + 1)
        if d == 0 or k % 10 == 9:
            assert np.array_equal(ref.digest(0, G), e.digest(0, G)), f"state after tick {k} (d = {d})"
    while pending:
        finish(pending.popleft())
    for t in range(ticks, ticks + d + 1):
        e.timers_due_wait(t % 4)
    assert np.array_equal(ref.digest(0, G), e.digest(0, G)), "state at the end"
    got = e.export_bulk(0, G)
    for g in range(0, G, 13):
        assert harness.state_bytes(got[g], F) == harness.state_bytes(o.export(g), F), f"group {g} (oracle)"
    roles = np.bincount(_table_bulk(e, G)["role"], minlength=3)
    print(f"d = {d}: due lists p50 {int(np.median(listed[1:]))} / max {max(listed[1:])}, rule lists p50 "
          f"{int(np.median(rule_listed[1:]))}, counts[3] p50 {int(np.median(counts))} / max {max(counts)}; "
          f"{tail_acks} acks of tail-position plans; roles {roles.tolist()}")
    assert sum(counts) > 20_000 and tail_acks > 1000, (sum(counts), tail_acks)
    assert roles[abi.ROLE_FOLLOWER] > 1000 and roles[abi.ROLE_LEADER] > 1000
    if d == 3:
        assert np.median(listed[1:]) < np.median(rule_listed[1:]), (np.median(listed[1:]), np.median(rule_listed[1:]))


def _sorted_inbox(ib: abi.Inbox, L: np.ndarray) -> tuple[abi.Inbox, np.ndarray]:
    """a positional inbox over the list L (ib.gids followed by a tail, ib padded for it) as the inbox over sorted(L), and the
    order that maps sorted positions back to L's"""
    order = np.argsort(L, kind="stable")
    s = abi.Inbox.__new__(abi.Inbox)
    s.__dict__.update(ib.__dict__)
    s.gids = np.ascontiguousarray(L[order], dtype=np.uint32)
    for name in ("op_meta", "op_nr", "op_ab", "op_cd", "op_e", "ev_meta", "ev_tn", "ev_el"):
        col = getattr(ib, name)
        if col is not None:
            setattr(s, name, np.ascontiguousarray(col[:, order]))
    return s, order


@pytest.mark.parametrize("flags", [EL, EL | PT])
def test_due_step_equals_the_sweep_step_over_its_list_on_the_storm(flags):
    """config #3 at R = 5: due steps over a fixed host list, with a cap of a third of counts[3] on the even steps (the due
    groups left over stay for the next) and above it on the odd ones; a twin engine takes the sweep step over
    sorted(gids u tail)."""
    G, R, rows = 16384, 5, 4
    F = R - 1
    cfg, init, w = model._storm_open(G, R, rows)
    e, ref = engine.Engine(cfg), engine.Engine(cfg)
    for s in (e, ref):
        s.open_bulk(0, init)
    A = np.sort(np.random.default_rng(5).choice(G, 2000, replace=False)).astype(np.uint32)
    prev, seen_over, seen_under = None, 0, 0
    for k in range(6):
        ib = workload.vote_inbox_host(w, k, prev, gids=A)
        ib.row_now = np.zeros(rows, np.int64)
        t0 = int(ib.op_nr["x"][ib.op_meta != 0].min()) if (ib.op_meta != 0).any() else workload.T0_MS
        ib.row_now[0] = t0 + 4000                                      # the storm's followers time out
        until = int(ib.row_now.max())
        t = _table_bulk(e, G)
        n_due_model = len(np.setdiff1d(np.flatnonzero(tm.due(t, until)), A))
        cap = max(1, n_due_model // 3) if k % 2 == 0 else n_due_model + 50
        want_tail, want_n = dm.tail(t, A, cap, until)
        ci = compact.encode_inbox(compact.due_inbox(ib, cap), None, None, elections=True, sweep=True)
        n = len(A) + cap
        cout = compact.CompactOutbox(rows, n, F, esc_cap=rows * n * F + 2 * rows * n)
        tail = e.step_compact_due(ci, cout, cap, slot=k % 4, reqs=ci.reqs, flags=flags)
        assert int(cout.counts[3]) == want_n and np.array_equal(tail, want_tail), f"step {k}: the tail"
        seen_over += want_n > cap; seen_under += want_n <= cap
        L = cout.gids
        si, order = _sorted_inbox(compact.due_inbox(ib, cap), L)
        cs = compact.encode_inbox(si, None, None, elections=True, sweep=True)
        rout = compact.CompactOutbox(rows, n, F, esc_cap=rows * n * F + 2 * rows * n, gids=si.gids)
        ref.step_compact(cs, rout, slot=k % 4, reqs=cs.reqs, flags=flags)
        got = compact.decode_outbox(cout, elections=True, prev_term=bool(flags & PT))
        want = compact.decode_outbox(rout, elections=True, prev_term=bool(flags & PT))
        back = np.empty(n, np.int64); back[order] = np.arange(n)         # position i of L is position back[i] of sorted(L)
        harness.assert_outbox_equal(_at(want, back), got, where=f"step {k}")
        assert np.array_equal(e.digest(0, G), ref.digest(0, G)), f"state after step {k}"
        prev = active.carry_outbox(got, L, A, G)
    assert seen_over >= 1 and seen_under >= 3, (seen_over, seen_under)   # the storm's first sweep holds most of its timeouts


def test_due_step_tail_is_the_due_query_list():
    """A due query and a due step over an empty host list, begun back to back in the same slot number, see one state: the
    query's list and next deadline equal the model's, counts[3] equals the query's n_due, and the tail is the query's first
    cap gids (cap below n_due), or the query's whole list followed by fillers (cap above it).  G is not a multiple of the
    selection's 256-group block."""
    G, R, rows = 5000, 3, 2
    F = R - 1
    cfg = abi.make_cfg(replicas=R, max_groups=G, max_rows=rows, entry_pool_cap=16)
    init = harness.init_array(G)
    init["rand_ms"] = 1 + np.random.default_rng(7).integers(0, 1000, G)      # followers' deadlines spread over 1 s
    e = engine.Engine(cfg)
    e.open_bulk(0, init)
    until = int(np.percentile(_table_bulk(e, G)["timer"], 40))
    ib = abi.Inbox(rows, G, F, with_ops=False, with_events=False, sweep=True)
    ib.row_now[0] = until
    host, q = np.zeros(0, np.uint32), np.zeros(G, np.uint32)

    def query_and_step(slot, cap_of):
        t = _table_bulk(e, G)
        want = np.flatnonzero(tm.due(t, until))
        cap = cap_of(len(want))
        ci = compact.encode_inbox(compact.due_inbox(tm.slice_inbox(ib, host), cap), None, None, sweep=True)
        cout = compact.CompactOutbox(rows, cap, F, esc_cap=rows * cap * F + 2 * rows * cap)
        e.timers_due_begin(slot, until, q)
        e.step_begin_compact_due(slot, host, cap, ci.sweep, ci.as_c(), None, cout.as_c())
        tail = e.step_wait_compact_due(slot)
        n_q, nxt = e.timers_due_wait(slot)
        assert n_q == len(want) and np.array_equal(q[:n_q], want), f"slot {slot}: the query's list"
        assert nxt == tm.next_deadline(t, until), f"slot {slot}: the query's next deadline"
        assert int(cout.counts[3]) == n_q and np.array_equal(tail, dm.tail(t, host, cap, until)[0]), f"slot {slot}: the tail"
        return q[:n_q].copy(), tail

    Q, tail = query_and_step(1, lambda n: n // 3)                       # the step fires a third of the due groups
    assert len(Q) > 300 and np.array_equal(tail, Q[:len(tail)])
    Q, tail = query_and_step(2, lambda n: n + 100)                      # ... and this one the rest
    assert len(Q) > 200 and np.array_equal(tail[:len(Q)], Q) and not np.isin(tail[len(Q):], Q).any()


def test_refusals_leave_the_slot_free():
    G, R, rows = 2048, 3, 2
    F = R - 1
    cfg = abi.make_cfg(replicas=R, max_groups=G, max_rows=rows, entry_pool_cap=rows * G * 50)
    e = engine.Engine(cfg)
    e.open_bulk(0, harness.init_array(G, terms=np.arange(G) % 7))
    harness.elect_all(e, workload.make_wl(0x5EED0002, 1, G, F))
    L = engine.lib()
    A = np.arange(0, G, 4, dtype=np.uint32)
    cap = 16
    n = len(A) + cap
    sweep = np.array([workload.T0_MS + 500, 0], np.int64)

    def inbox():
        ib = tm.slice_inbox(abi.Inbox(rows, G, F, ent_cap=1, sweep=True), A)
        ib.row_now = sweep.copy()
        return compact.due_inbox(ib, cap)

    keep = {}                                                            # what a begun step writes at its wait, per slot

    def begin(slot, ci, reqs=None, n_host=len(A), cap_=cap, sw=sweep, gids=A):
        cout = compact.CompactOutbox(rows, n, F, esc_cap=rows * n * F + 2 * rows * n)
        tail = np.zeros(max(cap_, 1), np.uint32)
        keep[slot] = (cout, tail, ci, reqs)                              # the wait writes counts and the tail into them
        return L.rafting_step_begin_compact_due(e._h, slot, n_host, gids.ctypes.data, cap_, sw.ctypes.data, C.byref(ci.as_c()),
                                                None if reqs is None else C.byref(reqs.as_c()), C.byref(cout.as_c()),
                                                tail.ctypes.data, 0)

    def rec_at(pos):
        req = np.zeros(1, abi.CREQ)
        req["slot"] = 1 * n + pos                                        # row 1 (not a sweep row), position pos
        req["meta"] = abi.creq_make(1, 0, 0)
        req["term"], req["d_prev_term"] = 100, 100
        return compact.CompactRequests(req)
    ci = compact.encode_inbox(inbox(), None, None, sweep=True)
    assert begin(0, ci, reqs=rec_at(len(A) + 2)) == -1                   # a request record at a tail position
    on_sweep = np.zeros(1, abi.CREQ); on_sweep["slot"] = 3
    assert begin(1, ci, reqs=compact.CompactRequests(on_sweep)) == -1    # a request record on the sweep row
    esc_ci = compact.encode_inbox(inbox(), None, None, sweep=True)
    esc_ci.esc = np.zeros(1, abi.CESC_IN); esc_ci.esc["slot"] = (n + len(A) + 1) * F   # a lane escape at a tail position
    assert begin(2, esc_ci) == -1
    assert begin(3, ci, sw=np.zeros(rows, np.int64)) == -1               # no sweep row
    assert begin(0, ci, cap_=0) == -1                                    # cap = 0
    assert begin(1, ci, cap_=G - len(A) + 1) == -5                       # not enough groups outside the list: RAFTING_E_CAPACITY
    bad = A.copy(); bad[[4, 5]] = bad[[5, 4]]
    assert begin(2, ci, gids=bad) == -1                                  # a decreasing host list
    for slot in range(4):                                                # every slot is free, and takes a due step
        assert begin(slot, ci, reqs=rec_at(1)) == 0
        e.step_wait_compact(slot)
        tail = keep[slot][1]
        assert len(np.unique(tail)) == cap and not np.isin(tail, A).any()


def test_due_native_through_the_jni_glue(tmp_path):
    from tests import jni_exec
    from tests.jni_exec import Buf, buf_of_array, buf_of_struct, fn
    Lj = jni_exec.build(str(tmp_path))
    if Lj is None:
        pytest.skip("no gcc")
    G, R, rows = 1024, 3, 2
    F = R - 1
    cfg = abi.make_cfg(replicas=R, max_groups=G, max_rows=rows, entry_pool_cap=rows * G * 50)
    o = binding.Oracle(cfg)
    Lj.fake_reset()
    h = fn(Lj, "create", C.c_int64, C.POINTER(Buf))(C.byref(buf_of_struct(cfg)))
    assert h != 0 and Lj.fake_throws() == 0, Lj.fake_thrown_message()
    init = harness.init_array(G, terms=np.arange(G) % 7)
    o.open_bulk(0, init)
    fn(Lj, "groupOpenBulk", None, C.c_int64, C.c_int32, C.c_int32, C.POINTER(Buf))(h, 0, G, C.byref(buf_of_array(init)))
    begin = fn(Lj, "stepBeginCompactDue", None, C.c_int64, C.c_int32, C.c_int32, C.POINTER(Buf), C.c_int32, C.POINTER(Buf),
               C.POINTER(Buf), C.POINTER(Buf), C.POINTER(Buf), C.POINTER(Buf), C.c_int32)
    wait = fn(Lj, "stepWaitCompact", None, C.c_int64, C.c_int32)
    t = tm.table([o.export(g) for g in range(G)])
    until = int(np.median(t["timer"]))
    due = np.flatnonzero(tm.due(t, until))
    cap = len(due) + 10
    ib = abi.Inbox(rows, G, F, with_ops=False, with_events=False, sweep=True)
    ib.row_now[0] = until
    want = o.step(ib)
    ci = compact.encode_inbox(compact.due_inbox(tm.slice_inbox(ib, np.zeros(0, np.uint32)), cap), None, None, sweep=True)
    cout = compact.CompactOutbox(rows, cap, F, esc_cap=rows * cap * F + 2 * rows * cap)
    tail = np.zeros(cap, np.uint32)
    begin(h, 1, 0, None, cap, C.byref(buf_of_array(ci.sweep)), C.byref(buf_of_struct(ci.as_c())), None,
          C.byref(buf_of_struct(cout.as_c())), C.byref(buf_of_array(tail)), 0)
    wait(h, 1)
    assert Lj.fake_throws() == 0, Lj.fake_thrown_message()
    assert int(cout.counts[3]) == len(due) and np.array_equal(tail[:len(due)], due)
    cout.gids = tail
    harness.assert_outbox_equal(_at(want, tail), compact.decode_outbox(cout), where="due step through the native")
    fn(Lj, "destroy", None, C.c_int64)(h)
