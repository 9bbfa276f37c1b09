"""Timers on the compact host path (`-m gpu`): rafting_step_begin_compact_sweep against the dense step with row_now, and
rafting_timers_due_begin / _wait against the exported state.

  * twin engines and the oracle in lock-step: the compact sweep step (compact.encode_inbox(sweep=True)) decodes to the dense
    engine's outbox and the oracle's, and leaves both engines in the same state — the R = 3 leader stream (pair_kernel),
    config #5 with its request list (class-sorted), the config #3 storm at R = 5 with flags 1 and 5 (election timeouts fired
    by the sweep), an active list of 4 096 of 64 K groups, sweep-only steps and multi-row steps with the sweep in row 0
  * the due list and the next deadline equal numpy over rafting_state_export_bulk at 1 M groups with mixed roles, closed
    groups and muted timers; until == a deadline; the cap overflow report; a query begun right after an un-waited step; four
    queries in flight; pinned and pageable output buffers
  * refusals leave the slot free; the new natives run through the stand-in JNIEnv"""
import ctypes as C

import numpy as np
import pytest

from oracle import binding
from rafting_b200 import abi, compact, engine, workload
from tests import compact_model as model
from tests import harness
from tests import timers_model as tm
from tests.compact_model import EL, PT

pytestmark = pytest.mark.gpu
U64 = np.uint64


def _strip(ib):
    """ib as a sweep-only step: no group op, no lane event"""
    ib.op_meta = ib.op_nr = ib.op_ab = ib.op_cd = ib.op_e = None
    ib.ev_meta = ib.ev_tn = ib.ev_el = None
    ib.ent_count = 0
    return ib


def _open(G, R, rows, kind):
    F = R - 1
    if kind == "storm":
        cfg, init, w = model._storm_open(G, R, rows)
    else:
        cfg = abi.make_cfg(replicas=R, max_groups=G, max_rows=rows, entry_pool_cap=rows * G * 50)
        init = harness.init_array(G, terms=np.arange(G) % 7)
        w = workload.make_wl(0x5EED0005 if kind == "mixed" else 0x5EED0002, rows, G, F)
    dense, comp, o = engine.Engine(cfg), engine.Engine(cfg), binding.Oracle(cfg)
    for s in (dense, comp, o):
        s.open_bulk(0, init)
    if kind != "storm":
        w1 = workload.make_wl(0x5EED0005, 1, G, F)
        want = harness.elect_all(o, w1)
        for e in (dense, comp):
            harness.assert_outbox_equal(want, harness.elect_all(e, w1), where="election")
    gen = {"storm": workload.vote_inbox_host, "mixed": workload.mixed_inbox_host, "leader": workload.leader_inbox_host}[kind]
    return cfg, dense, comp, o, w, gen


CASES = {   # kind, G, R, rows, flags, active-list size
    "leader_r3": ("leader", 16384, 3, 4, 0, 0),
    "config5_reqs": ("mixed", 16384, 3, 4, 0, 0),
    "config3_storm_f1": ("storm", 16384, 5, 4, EL, 0),
    "config3_storm_f5": ("storm", 16384, 5, 4, EL | PT, 0),
    "leader_active_4096_of_64k": ("leader", 65536, 3, 4, 0, 4096),
}


@pytest.mark.parametrize("case", sorted(CASES))
def test_compact_sweep_step_equals_the_dense_step(case):
    kind, G, R, rows, flags, n_act = CASES[case]
    F = R - 1
    cfg, dense, comp, o, w, gen = _open(G, R, rows, kind)
    A = np.sort(np.random.default_rng(7).choice(G, n_act, replace=False)).astype(np.uint32) if n_act else None
    prev, nxt, fired = None, None, 0
    for k in range(8):
        ib = gen(w, k, prev, gids=A)
        t = int(ib.op_nr["x"][ib.op_meta != 0].min()) if ib.op_meta is not None and (ib.op_meta != 0).any() else workload.T0_MS + 10 * k
        ib.row_now = np.zeros(rows, np.int64)
        ib.row_now[0] = t + (4000 if kind == "storm" else 60 * k)        # the storm's followers time out; leaders heartbeat
        if k % 4 == 3:
            ib.row_now[2] = ib.row_now[0] + 100                          # a second sweep row
        if k % 4 == 2:
            ib = _strip(ib)                                              # a sweep-only step
        want = o.step(ib, threads=8)
        harness.assert_outbox_equal(want, dense.step(ib), where=f"dense step {k}")
        ci = compact.encode_inbox(ib, **(nxt or dict(tags=None, sent_term=None)), elections=bool(flags & EL), sweep=True)
        if k % 4 == 2:
            assert ci.op_c is None and ci.ev_c is None and ci.reqs is None
        n = ib.n
        cout = compact.CompactOutbox(rows, n, F, esc_cap=rows * n * F + 2 * rows * n, gids=A)
        comp.step_compact(ci, cout, slot=k % 4, reqs=ci.reqs, flags=flags)
        got = compact.decode_outbox(cout, elections=bool(flags & EL), prev_term=bool(flags & PT))
        harness.assert_outbox_equal(want, got, where=f"compact sweep step {k}")
        sw = ib.row_now != 0
        fired += int((want.plan_meta[sw] != 0).sum() + (want.ballot_meta[sw] != 0).sum())
        nxt, prev = model.next_of(want, cout), want
    assert fired > 100, fired
    a, b = dense.export_bulk(0, G), comp.export_bulk(0, G)
    for g in range(G):
        assert harness.state_bytes(a[g], F) == harness.state_bytes(b[g], F), f"group {g}"
    for g in range(0, G, 7):
        assert harness.state_bytes(b[g], F) == harness.state_bytes(o.export(g), F), f"group {g} (oracle)"


def _table_bulk(e, G, chunk=65536):
    """timer / role / alive of every group through rafting_state_export_bulk, read from the structs' bytes"""
    out = dict(timer=np.zeros(G, np.int64), role=np.zeros(G, np.int64), alive=np.zeros(G, np.int64))
    size = C.sizeof(abi.GroupState)
    for first in range(0, G, chunk):
        n = min(chunk, G - first)
        raw = np.frombuffer(e.export_bulk(first, n), dtype=np.uint8).reshape(n, size)
        for name, dt in (("timer", np.int64), ("role", np.uint32), ("alive", np.uint32)):
            off = getattr(abi.GroupState, name).offset
            out[name][first:first + n] = raw[:, off:off + np.dtype(dt).itemsize].copy().view(dt)[:, 0]
    return out


def _mixed_million():
    """config #4's size on one GPU: 1 M groups through two steps of the config #3 storm (followers, candidates, leaders), then
    muted timers (a stale installSnapshot at every 13th group that is a follower) and closed groups"""
    G, R, rows = 1 << 20, 3, 2
    cfg, init, w = model._storm_open(G, R, rows)
    e = engine.Engine(cfg)
    e.open_bulk(0, init)
    prev = None
    for k in range(2):
        prev = e.step(workload.vote_inbox_host(w, k, prev))
    t = _table_bulk(e, G)
    ib = abi.Inbox(1, G, R - 1, ent_cap=1)
    st = np.zeros(G, np.int64)
    st_term = np.array(prev.current_term, np.int64)
    g = np.flatnonzero((np.arange(G) % 13 == 0) & (t["role"] == abi.ROLE_FOLLOWER) & (st_term > 0))
    ib.op_meta[0, g] = abi.op_make(abi.OP_IS_REQUEST, 0)
    ib.op_nr["x"][0, g] = workload.T0_MS + 500
    ib.op_ab["x"][0, g] = st_term[g] - 1
    e.step(ib)
    for gid in range(11, G, 4099):
        e.close_group(gid)
    return e, G


@pytest.fixture(scope="module")
def million():
    e, G = _mixed_million()
    yield e, G
    e.close()


def test_due_list_matches_the_exported_state_at_a_million_groups(million):
    import torch
    e, G = million
    t = _table_bulk(e, G)
    roles = np.bincount(t["role"], minlength=3)
    assert (roles > 1000).sum() >= 2, roles                               # mixed roles
    assert (t["alive"] == 0).sum() > 200 and ((t["alive"] != 0) & (t["timer"] == tm.I64MAX)).sum() > 0, "closed groups, muted timers"
    armed = np.sort(t["timer"][(t["alive"] != 0) & (t["timer"] > 0) & (t["timer"] != tm.I64MAX)])
    pinned = torch.zeros(G, dtype=torch.int32).pin_memory()
    for until in (int(armed[len(armed) // 10]), int(armed[len(armed) // 2]), int(armed[len(armed) // 2]) - 1, int(armed[-1])):
        want = np.flatnonzero(tm.due(t, until))
        got, nxt = e.timers_due(until)                                   # pageable buffer: the staged copy
        assert np.array_equal(got, want) and nxt == tm.next_deadline(t, until), until
        e.timers_due_begin(1, until, pinned.data_ptr(), G)               # pinned: the device writes the caller's buffer
        n, nxt2 = e.timers_due_wait(1)
        assert n == len(want) and nxt2 == nxt
        assert np.array_equal(pinned.numpy()[:n].view(np.uint32), want)
        assert (t["timer"][want] == until).any() or until != int(armed[len(armed) // 2])
    # cap overflow: the count is the whole count, the first cap gids are written, nothing past them
    until = int(armed[len(armed) // 2])
    want = np.flatnonzero(tm.due(t, until))
    cap = len(want) // 3
    out = np.full(cap + 8, 0xFFFFFFFF, np.uint32)
    e.timers_due_begin(2, until, out, cap)
    n, _ = e.timers_due_wait(2)
    assert n == len(want) and np.array_equal(out[:cap], want[:cap]) and (out[cap:] == 0xFFFFFFFF).all()
    # four queries in flight at once
    us = [int(armed[q * len(armed) // 5]) for q in range(1, 5)]
    bufs = [np.zeros(G, np.uint32) for _ in us]
    for s, (u, b) in enumerate(zip(us, bufs)):
        e.timers_due_begin(s, u, b)
    with pytest.raises(engine.RaftingError):
        e.timers_due_begin(0, us[0], bufs[0])                            # slot 0 is taken
    for s, (u, b) in enumerate(zip(us, bufs)):
        n, nxt = e.timers_due_wait(s)
        w = np.flatnonzero(tm.due(t, u))
        assert n == len(w) and np.array_equal(b[:n], w) and nxt == tm.next_deadline(t, u)
    n, nxt = e.timers_due_begin(3, 0, None) or e.timers_due_wait(3)      # cap 0: the count only
    assert n == int(tm.due(t, 0).sum())


def test_a_query_sees_the_step_begun_before_it():
    G, R, rows = 65536, 3, 2
    cfg = abi.make_cfg(replicas=R, max_groups=G, max_rows=rows, entry_pool_cap=rows * G * 50)
    e = engine.Engine(cfg)
    e.open_bulk(0, harness.init_array(G, terms=np.arange(G) % 7))
    harness.elect_all(e, workload.make_wl(0x5EED0002, 1, G, R - 1))
    t = _table_bulk(e, G)
    until = int(np.median(t["timer"]))
    ib = _strip(abi.Inbox(rows, G, R - 1, sweep=True))
    ib.row_now[0] = until                                                 # fires the heartbeats due at `until`
    ci = compact.encode_inbox(ib, None, None, sweep=True)
    cout = compact.CompactOutbox(rows, G, R - 1, esc_cap=4096)
    e.step_begin_compact_sweep(0, ci.sweep, ci.as_c(), None, cout.as_c())
    out = np.zeros(G, np.uint32)
    e.timers_due_begin(0, until, out)                                     # the step has not been waited for
    n, _ = e.timers_due_wait(0)
    e.step_wait_compact(0)
    after = _table_bulk(e, G)
    assert int(tm.due(t, until).sum()) > 1000 and n == int(tm.due(after, until).sum()) == 0


def test_refusals_leave_the_slot_free():
    G, R, rows = 2048, 3, 2
    F = R - 1
    cfg, dense, comp, o, w, gen = _open(G, R, rows, "mixed")
    L = engine.lib()
    ib = abi.Inbox(rows, G, F, ent_cap=1)
    ib.ae_request(1, 5, workload.T0_MS, leader=0, term=100, prev_index=0, prev_term=0)   # a record at row 1
    ci = compact.encode_inbox(ib, None, None)
    assert ci.reqs is not None and len(ci.reqs.req) == 1
    cout = compact.CompactOutbox(rows, G, F, esc_cap=rows * G * F + 2 * rows * G)
    row_of_first = int(ci.reqs.req["slot"][0]) // G
    on_req = np.zeros(rows, np.int64); on_req[row_of_first] = workload.T0_MS
    A = np.arange(0, G, 3, dtype=np.uint32)
    bad = A.copy(); bad[[4, 5]] = bad[[5, 4]]
    zero = np.zeros(rows, np.int64)

    def begin(slot, sweep, gids=None, n=None, flags=0):
        return L.rafting_step_begin_compact_sweep(comp._h, slot, len(gids) if n is None and gids is not None else (n or 0),
                                                  None if gids is None else gids.ctypes.data, sweep.ctypes.data,
                                                  C.byref(ci.as_c()), C.byref(ci.reqs.as_c()), C.byref(cout.as_c()), flags)
    assert begin(0, on_req) == -1                                         # a request record on a sweep row
    assert begin(1, zero, gids=bad) == -1                                 # a decreasing list
    assert begin(2, zero, gids=A, n=0) == -1                              # an empty list
    assert begin(3, zero, flags=2) == -1                                  # an unknown flag
    assert L.rafting_step_begin_compact_sweep(comp._h, 4, 0, None, zero.ctypes.data, C.byref(ci.as_c()), None,
                                              C.byref(cout.as_c()), 0) == -1   # a bad slot
    assert L.rafting_timers_due_begin(comp._h, 4, 0, None, 0) == -1
    assert L.rafting_timers_due_wait(comp._h, 0, None, None) == -1      # nothing in flight
    for slot in range(4):                                                 # every slot is free and the next steps are exact
        ib = workload.mixed_inbox_host(w, slot, None if slot == 0 else want)
        want = o.step(ib, threads=8)
        ci = compact.encode_inbox(ib, None, None, sweep=True)
        cout = compact.CompactOutbox(rows, G, F, esc_cap=rows * G * F + 2 * rows * G)
        comp.step_compact(ci, cout, slot=slot, reqs=ci.reqs)
        harness.assert_outbox_equal(want, compact.decode_outbox(cout), where=f"slot {slot}")


def test_sweep_and_due_natives_through_the_jni_glue(tmp_path):
    from tests import jni_exec
    from tests.jni_exec import Buf, buf_of_array, buf_of_struct, fn
    L = jni_exec.build(str(tmp_path))
    if L is None:
        pytest.skip("no gcc")
    G, R, rows = 1024, 3, 2
    F = R - 1
    cfg = abi.make_cfg(replicas=R, max_groups=G, max_rows=rows, entry_pool_cap=rows * G * 50)
    o = binding.Oracle(cfg)
    L.fake_reset()
    h = fn(L, "create", C.c_int64, C.POINTER(Buf))(C.byref(buf_of_struct(cfg)))
    assert h != 0 and L.fake_throws() == 0, L.fake_thrown_message()
    init = harness.init_array(G, terms=np.arange(G) % 7)
    o.open_bulk(0, init)
    fn(L, "groupOpenBulk", None, C.c_int64, C.c_int32, C.c_int32, C.POINTER(Buf))(h, 0, G, C.byref(buf_of_array(init)))
    begin = fn(L, "stepBeginCompactSweep", None, C.c_int64, C.c_int32, C.c_int32, C.POINTER(Buf), C.POINTER(Buf), C.POINTER(Buf),
               C.POINTER(Buf), C.POINTER(Buf), C.c_int32)
    wait = fn(L, "stepWaitCompact", None, C.c_int64, C.c_int32)
    due_begin = fn(L, "timersDueBegin", None, C.c_int64, C.c_int32, C.c_int64, C.POINTER(Buf), C.c_int32)
    due_wait = fn(L, "timersDueWait", None, C.c_int64, C.c_int32, C.POINTER(jni_exec.Longs))
    t = tm.table([o.export(g) for g in range(G)])
    until = int(np.median(t["timer"]))
    out = np.zeros(G, np.uint32)
    due_begin(h, 2, until, C.byref(buf_of_array(out)), G)
    arr = np.zeros(2, np.int64)
    due_wait(h, 2, C.byref(jni_exec.Longs(2, arr.ctypes.data_as(C.POINTER(C.c_int64)))))
    assert L.fake_throws() == 0, L.fake_thrown_message()
    want = np.flatnonzero(tm.due(t, until))
    assert arr[0] == len(want) and np.array_equal(out[:len(want)], want) and arr[1] == tm.next_deadline(t, until)
    ib = _strip(abi.Inbox(rows, G, F, sweep=True))
    ib.row_now[0] = until
    want_o = o.step(ib)
    ci = compact.encode_inbox(ib, None, None, sweep=True)
    A = np.arange(G, dtype=np.uint32)
    cout = compact.CompactOutbox(rows, G, F, esc_cap=rows * G * F + 2 * rows * G, gids=A)
    begin(h, 1, G, C.byref(buf_of_array(A)), C.byref(buf_of_array(ci.sweep)), C.byref(buf_of_struct(ci.as_c())), None,
          C.byref(buf_of_struct(cout.as_c())), 0)
    wait(h, 1)
    assert L.fake_throws() == 0, L.fake_thrown_message()
    harness.assert_outbox_equal(want_o, compact.decode_outbox(cout), where="compact sweep step through the natives")
    fn(L, "destroy", None, C.c_int64)(h)


def _positional(o: abi.Outbox, L: np.ndarray) -> abi.Outbox:
    """the whole-shard outbox o restricted to the list L, by position (the COMPACT_GROUPS shape)"""
    p = abi.Outbox(o.rows, len(L), o.F, len(L))
    g = L.astype(np.int64)
    for name, _, _ in abi.Outbox.ROW_COLS:
        getattr(p, name)[...] = getattr(o, name)[:, g]
    for name, _ in abi.Outbox.GROUP_COLS:
        getattr(p, name)[...] = getattr(o, name)[g]
    return p


@pytest.mark.parametrize("d", [0, 3])
def test_closed_loop_on_due_lists_matches_whole_shard_sweeps(d):
    """A 64 K x 3 shard for 320 ticks of tests/timers_model.Peers (followers kept by heartbeats, leaderless groups electing, a
    leader lost at tick 150 and a second election wave), two ways: the reference engine takes dense whole-shard steps with a
    sweep row; the candidate engine takes compact active sweep steps over the pipelining rule's lists, d steps in flight
    (d = 3: four slots), each list built from a due query begun right after step k-d.  Every waited step's decoded outbox
    equals the reference's at the listed groups, the reference did nothing at the others, both engines' states are equal
    (digest of every group; every tick at d = 0, every 10th and the last at d = 3, so that steps stay in flight on the device),
    and at the end both equal the oracle."""
    import torch
    from collections import deque
    from tests import compact_active_model as active
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
    wants, terms = [], init["term"].astype(np.int64)
    lists, events, steps = {}, {}, {}
    pending = deque()
    listed, due_hb, due_ballots = [], 0, 0

    def begin_query(t):
        e.timers_due_begin(t % 4, P.now(t), bufs[t % 4].data_ptr(), G)

    def finish(j):
        e.step_wait_compact(j % 4)
        ci, cout, L = steps[j]
        got = compact.decode_outbox(cout)
        harness.assert_outbox_equal(_positional(wants[j], L), got, where=f"step {j} (d = {d})")
        steps[j] = (None, cout, L)

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
        n_due, _ = e.timers_due_wait(k % 4)
        Q = bufs[k % 4].numpy()[:n_due].view(np.uint32).astype(np.int64)
        events[k] = tm.event_gids(ib)
        flight = [events[j] for j in pending]
        L = np.union1d(np.union1d(Q, events[k]), np.concatenate(flight) if flight else np.zeros(0, np.int64)).astype(np.uint32)
        # what the reference did outside the list: nothing
        out_of_list = np.ones(G, bool); out_of_list[L.astype(np.int64)] = False
        assert not want.rep_meta[:, out_of_list].any() and not want.plan_meta[:, out_of_list].any() and \
            not want.ballot_meta[:, out_of_list].any(), f"the whole-shard step acted on an unlisted group, tick {k}"
        fired = (want.plan_meta[0] != 0).any(axis=1) | (want.ballot_meta[0] != 0)
        only_due = np.zeros(G, bool); only_due[Q] = True
        only_due[events[k]] = False
        for f_ in flight:
            only_due[f_] = False
        due_hb += int((fired & only_due & (want.plan_meta[0] != 0).any(axis=1)).sum())
        due_ballots += int((fired & only_due & (want.ballot_meta[0] != 0)).sum())
        listed.append(len(L))
        if len(L):
            ai = tm.slice_inbox(ib, L)
            tags = np.full((rows, len(L), F), abi.CTAG_NONE, np.uint8)
            sent_term, sent_inc = np.zeros(len(L), np.int64), np.zeros(len(L), np.uint32)
            j = k - P.DELAY
            if j in steps and steps[j][0] is None:                   # the step whose plans these acks answer (waited)
                _, cj, Lj = steps[j]
                p = active.positions(Lj, L, G)
                has, q = p >= 0, np.maximum(p, 0)
                tp = cj.tags(rpc_only=True)
                for r in range(2):
                    tags[r + 1][has] = tp[r][q[has]]
                sent_term[has], sent_inc[has] = cj.current_term[q[has]], cj.incarnation[q[has]]
            ci = compact.encode_inbox(ai, tags, sent_term, sent_inc, sweep=True)
            n = len(L)
            cout = compact.CompactOutbox(rows, n, F, esc_cap=rows * n * F + 2 * rows * n, gids=L)
            e.step_begin_compact_sweep(k % 4, ci.sweep, ci.as_c(), None if ci.reqs is None else ci.reqs.as_c(), cout.as_c(),
                                       gids=L)
            steps[k] = (ci, cout, L)
            pending.append(k)
        steps.pop(k - P.DELAY - 1, None)
        begin_query(k + d + 1)                                           # sees every step up to k
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
    print(f"d = {d}: groups listed per step min {min(listed[1:])} / p50 {int(np.median(listed[1:]))} / max {max(listed[1:])} "
          f"of {G}; fired by the due list alone: {due_hb} heartbeats, {due_ballots} ballots; roles at the end {roles.tolist()}")
    assert due_hb > 10_000 and due_ballots > 10_000, (due_hb, due_ballots)    # heartbeats and two election waves
    assert roles[abi.ROLE_FOLLOWER] > 1000 and roles[abi.ROLE_LEADER] > 1000
    assert np.median(listed[1:]) < G
