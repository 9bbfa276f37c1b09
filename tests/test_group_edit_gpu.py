"""Group edits in step-stream order (`-m gpu`): rafting_group_edit_begin opens, restarts and closes groups while steps are in
flight, and leaves each gid exactly as the synchronous calls would at the same point of the stream.

  * a 64 K x 3 closed loop of tests/timers_model.Peers on compact due steps at d = 3 (four slots in flight at every edit),
    256 edits every 10 ticks: every waited outbox equals the dense reference's (synchronous calls after a drain) at the
    listed groups, the digests are equal at every tick but the ones right before an edit (a digest drains the stream, and
    the edit is to meet steps in flight), and at the end every group equals the oracle's
  * ordering against a step begun before and one begun after the edit, with rafting_group_open refused meanwhile
  * a due query begun after an OPEN lists the gid from its restored deadline on; state images after edits
  * tags: a gid closed and reopened while its lanes hold unanswered tags starts every new life at tag 0 through
    rafting_group_edit_begin, and runs out of tags after a few lives through the synchronous calls; both engines' compact
    outboxes (whole-shard and active sweep steps) equal tests/compact_model.py's, with the gid's lane bits zeroed at the edit
    on the first
  * each malformed record is refused with nothing enqueued
  * per-group restarts inside a live node of the cluster model, through rafting_group_edit_begin, against the oracle
  * the JNI native, through the stand-in JNIEnv, in lock-step with the oracle"""
import ctypes as C

import numpy as np
import pytest

from oracle import binding
from rafting_b200 import abi, compact, engine, workload
from rafting_b200.engine import RaftingError, edit_close, edit_open
from tests import compact_model as cm
from tests import edit_pump as ep
from tests import harness
from tests import timers_model as tm

pytestmark = pytest.mark.gpu

E_INVAL, E_CAPACITY, E_BUSY = -1, -5, -7


def _at(o: abi.Outbox, where: np.ndarray) -> abi.Outbox:
    p = abi.Outbox(o.rows, len(where), o.F, len(where))
    g = where.astype(np.int64)
    for name, _, _ in abi.Outbox.ROW_COLS:
        getattr(p, name)[...] = getattr(o, name)[:, g]
    for name, _ in abi.Outbox.GROUP_COLS:
        getattr(p, name)[...] = getattr(o, name)[g]
    return p


def test_edits_with_four_steps_in_flight_equal_the_synchronous_calls():
    ticks, G, F = 200, ep.G, ep.F
    o = binding.Oracle(ep.make_cfg())
    S = ep.Stream(k_edits=256, oracle=o)
    A = ep.DuePump(S, d=3, mode="edit")
    waited, digests, kinds = [0], [0], {1: 0, 2: 0}

    def on_wait(j, cout):
        harness.assert_outbox_equal(_at(S.wants[j], cout.gids), compact.decode_outbox(cout), where=f"step {j}")
        waited[0] += 1

    def on_tick(k):
        if k in S.edits:
            for kd in (abi.EDIT_OPEN, abi.EDIT_CLOSE):
                kinds[kd] += int((S.edits[k]["kind"] == kd).sum())
        if k + 1 not in S.edits:
            assert np.array_equal(S.ref.digest(0, G), A.e.digest(0, G)), f"state after tick {k}"
            digests[0] += 1

    A.run(ticks, on_wait=on_wait, on_tick=on_tick)
    assert waited[0] == ticks and digests[0] > 150
    assert np.array_equal(S.ref.digest(0, G), A.e.digest(0, G)), "state at the end"
    got = A.e.export_bulk(0, G)
    for g in range(G):
        assert harness.state_bytes(got[g], F) == harness.state_bytes(o.export(g), F), f"group {g} (oracle)"
    runs = np.concatenate([r["n_runs"] for r in S.edits.values()])
    assert kinds[abi.EDIT_OPEN] > 1000 and kinds[abi.EDIT_CLOSE] > 1000 and runs.max() == abi.TERM_RUNS, (kinds, runs.max())
    roles = np.bincount(np.array([s.role for s in got]), minlength=3)
    assert roles[abi.ROLE_LEADER] > 1000, roles


def _small(G=64, R=3):
    cfg = abi.make_cfg(replicas=R, max_groups=G, max_rows=2)
    init = harness.init_array(G, terms=np.full(G, 5))
    init["now_ms"] = workload.T0_MS
    init["rand_ms"] = 1_000_000
    return cfg, init


def _sweep_inbox(G, F, now):
    ib = abi.Inbox(1, G, F, sweep=True)
    ib.row_now[0] = now
    return ib


def test_an_edit_sits_between_the_steps_begun_before_and_after_it():
    cfg, init = _small()
    G, F, g = cfg.max_groups, cfg.replicas - 1, 17
    e = engine.Engine(cfg)
    e.open_bulk(0, init)
    ib = _sweep_inbox(G, F, workload.T0_MS + 10)
    o1, o2 = abi.Outbox(1, G, F, G), abi.Outbox(1, G, F, G)
    e.step_begin_host(0, ib.as_c(), o1.as_c())
    with pytest.raises(RaftingError) as x:
        e.open_group(g, term=9)
    assert x.value.rc == E_BUSY
    e.group_edit_begin([edit_close(g - 1), edit_open(g, term=9, ballot=1, now_ms=workload.T0_MS, rand_ms=1_000_000)])
    e.step_begin_host(1, ib.as_c(), o2.as_c())
    e.step_wait_slot(0)
    e.step_wait_slot(1)
    assert o1.current_term[g] == 5 and o2.current_term[g] == 9
    st = e.export(g)
    assert st.alive == 1 and st.current_term == 9 and st.voted_for == 1 and st.incarnation == 1
    assert e.export(g - 1).alive == 0 and e.export(g + 1).current_term == 5


def test_due_query_sees_the_restored_deadline_and_images_match_the_synchronous_calls(tmp_path):
    cfg, init = _small()
    G, F, g, T = cfg.max_groups, cfg.replicas - 1, 33, workload.T0_MS + 500
    a, b = engine.Engine(cfg), engine.Engine(cfg)
    for s in (a, b):
        s.open_bulk(0, init)
    recs = np.array([edit_open(3, runs=[(1, 1), (4, 2), (9, 4)], term=6, ballot=0, last_index=12, last_term=4, now_ms=T, rand_ms=77),
                     edit_close(8),
                     edit_open(g, term=6, now_ms=T, rand_ms=50)], dtype=abi.GROUP_EDIT)
    ib, out = _sweep_inbox(G, F, workload.T0_MS + 10), abi.Outbox(1, G, F, G)        # alive until the wait: the copies read them
    a.step_begin_host(0, ib.as_c(), out.as_c())                                          # a step in flight
    a.group_edit_begin(recs)
    bufs = [np.zeros(G, np.uint32) for _ in range(2)]
    a.timers_due_begin(1, T + 49, bufs[0])
    a.timers_due_begin(2, T + 50, bufs[1])
    a.step_wait_slot(0)
    for q, (slot, want) in enumerate(((1, False), (2, True))):
        n, _ = a.timers_due_wait(slot)
        assert (g in bufs[q][:n]) == want, (slot, bufs[q][:n])
    b.step(ib)
    ep.apply_sync(b, recs)
    assert np.array_equal(a.digest(0, G), b.digest(0, G))
    assert a.log_term(3, 5) == 2 and a.log_term(3, 12) == 4
    # dense steps and a state image after the edits
    for k in range(3):
        ib = _sweep_inbox(G, F, T + 100 * k)
        harness.assert_outbox_equal(a.step(ib), b.step(ib), where=f"dense step {k}")
    a.group_edit_begin([edit_close(3)])
    b.close_group(3)
    pa, pb = str(tmp_path / "a.img"), str(tmp_path / "b.img")
    a.state_save(pa), b.state_save(pb)
    c, d = engine.Engine(cfg), engine.Engine(cfg)
    c.state_load(pa), d.state_load(pb)
    assert np.array_equal(c.digest(0, G), d.digest(0, G)) and np.array_equal(c.digest(0, G), b.digest(0, G))


def test_a_reopened_gid_starts_at_tag_0_and_the_synchronous_reopen_leaks_its_tags():
    """gid 0 of a 3-node shard (tests/timers_model.Peers: its election timer fires, the peers grant the votes) becomes leader
    in every life and takes a client write each tick.  The AppendEntries those writes start (row 2) are never answered, so
    its lanes take tags until IN_FLIGHT_LIMIT stops the plans.  Every
    LIFE ticks it is reopened: on engine A with rafting_group_edit_begin, on engine B with the synchronous calls.  Both run
    the same stream of compact sweep steps, whole-shard and active by turns."""
    G, R, rows, LIFE, lives = 8, 3, 3, 60, 4
    F = R - 1
    cfg = abi.make_cfg(replicas=R, max_groups=G, max_rows=rows, entry_pool_cap=64, heartbeat_ms=10, election_ms=50)
    init = harness.init_array(G, terms=1 + np.arange(G) % 5)
    init["now_ms"] = workload.T0_MS
    o, A, B = binding.Oracle(cfg), engine.Engine(cfg), engine.Engine(cfg)
    for s_ in (o, A, B):
        s_.open_bulk(0, init)
    P = tm.Peers(G, rows=rows, lost_at=10**9, t0=workload.T0_MS)
    model = {"A": cm.InFlight(G, F), "B": cm.InFlight(G, F)}
    sent = {"A": {}, "B": {}}
    wants, terms, edited_at = [], init["term"].astype(np.int64), np.full(G, -10**9, np.int64)
    esc_cap = rows * G * F + 2 * rows * G
    held = {"A": [], "B": []}                     # tags gid 0's lanes hold when a life ends
    firsts = {"A": [], "B": []}                   # per life and lane: the tag of the first AppendEntries
    untagged = {"A": [0] * lives, "B": [0] * lives}
    life, first_seen = 0, {"A": set(), "B": set()}
    for k in range(LIFE * lives):
        if k > 0 and k % LIFE == 0:
            for name in ("A", "B"):
                held[name].append([bin(int(b)).count("1") for b in model[name].bits[0]])
            kw = dict(term=int(o.export(0).current_term), now_ms=P.now(k - 1), rand_ms=30)
            A.group_edit_begin([edit_open(0, **kw)])
            model["A"].bits[0] = 0                                      # what the edit does to the in-flight table
            ep.apply_sync(B, np.array([edit_open(0, **kw)], dtype=abi.GROUP_EDIT))
            ep.apply_sync(o, np.array([edit_open(0, **kw)], dtype=abi.GROUP_EDIT))
            edited_at[0] = k
            life, first_seen = life + 1, {"A": set(), "B": set()}
        ib = P.inbox(k, wants[k - P.DELAY] if k >= P.DELAY else None, terms)
        ib.submit(2, 0, P.now(k), count=1)          # a client write each tick; the peers answer plans of rows 0 and 1 only
        ep.drop_replies(ib, k, edited_at, P.DELAY)
        want = o.step(ib)
        wants.append(want)
        start_terms, terms = terms, want.current_term.copy()
        epoch = cm.oracle_epoch(o, G)
        pk = (want.plan_meta[:, 0, :] & np.uint64(0xF)).astype(np.int64)
        plans = (pk == abi.PLAN_AE) | (pk == abi.PLAN_IS)
        for name, e in (("A", A), ("B", B)):
            nx = sent[name].get(k - P.DELAY)
            ci = compact.encode_inbox(ib, *(nx if nx else (None, None, None)), sweep=True)
            gids = np.arange(G, dtype=np.uint32) if k % 2 else None
            cout = compact.CompactOutbox(rows, G, F, esc_cap=esc_cap, gids=gids)
            e.step_begin_compact_sweep(0, ci.sweep, ci.as_c(), None if ci.reqs is None else ci.reqs.as_c(), cout.as_c(), gids=gids)
            e.step_wait_compact(0)
            where = f"engine {name}, tick {k}"
            harness.assert_outbox_equal(want, compact.decode_outbox(cout), where=where)
            cm.unpack(ci, start_terms, model[name])                      # the acks free their tags
            m = cm.pack(want, epoch, model[name], esc_cap, replies=ci.reqs is not None)
            assert np.array_equal(cout.plan_c, m.plan_c), f"plan_c differs from the model, {where}"
            assert np.array_equal(cout.counts, m.counts) and cm._sorted_esc(cout) == cm._sorted_esc(m), f"escapes, {where}"
            sent[name][k] = (cout.tags(rpc_only=True), cout.current_term.copy(), cout.incarnation.copy())
            sent[name].pop(k - P.DELAY - 1, None)
            tg = cout.tags()[:, 0, :]
            untagged[name][life] += int((plans & (tg == abi.CTAG_NONE)).sum())
            for r, f in np.argwhere(plans):
                if f not in first_seen[name]:
                    first_seen[name].add(f)
                    firsts[name].append((life, int(f), int(tg[r, f])))
    print("tags held at the end of each life:", held, "untagged plans per life:", untagged)
    assert all(min(h) >= 16 for h in held["A"]), held              # every life ended with its lanes full of unanswered tags
    assert {lf for lf, _, _ in firsts["A"]} == set(range(lives)), firsts["A"]
    assert all(t == 0 for lf, _, t in firsts["A"]), firsts["A"]
    assert untagged["A"] == [0] * lives, untagged
    assert untagged["B"][0] == 0 and sum(untagged["B"][1:]) > 0, untagged
    assert any(t != 0 for lf, _, t in firsts["B"] if lf > 0), firsts["B"]


BAD = [
    ("gid beyond max_groups", lambda G: [edit_open(G)], E_CAPACITY),
    ("decreasing gid", lambda G: [edit_open(5), edit_close(4)], E_INVAL),
    ("repeated gid", lambda G: [edit_open(5), edit_close(5)], E_INVAL),
    ("unknown kind", lambda G: [dict_kind(edit_open(5), 3)], E_INVAL),
    ("bad ballot", lambda G: [edit_open(5, ballot=3)], E_INVAL),
    ("first_index rule", lambda G: [edit_open(5, epoch_index=4, first_index=9, last_index=12, last_term=1)], E_INVAL),
    ("runs do not start at first_index", lambda G: [edit_open(5, last_index=12, last_term=2, runs=[(2, 1), (5, 2)])], E_INVAL),
    ("last run's term is not last_term", lambda G: [edit_open(5, last_index=12, last_term=3, runs=[(1, 1), (5, 2)])], E_INVAL),
    ("runs outside the log", lambda G: [edit_open(5, last_index=12, last_term=2, runs=[(1, 1), (13, 2)])], E_INVAL),
    ("runs without a term change", lambda G: [edit_open(5, last_index=12, last_term=1, runs=[(1, 1), (5, 1)])], E_INVAL),
    ("runs over an empty log", lambda G: [edit_open(5, runs=[(1, 0)])], E_INVAL),
    ("n_runs > 8", lambda G: [n_runs(edit_open(5, last_index=12, last_term=1, runs=[(1, 1)]), 9)], E_CAPACITY),
]


def dict_kind(r, kind):
    r["kind"] = kind
    return r


def n_runs(r, n):
    r["n_runs"] = n
    return r


def test_each_malformed_record_is_refused_with_nothing_enqueued():
    cfg, init = _small()
    G, F = cfg.max_groups, cfg.replicas - 1
    a, b = engine.Engine(cfg), engine.Engine(cfg)
    for s in (a, b):
        s.open_bulk(0, init)
    before = a.digest(0, G)
    good = edit_open(1, term=7)
    for what, make, rc in BAD:
        with pytest.raises(RaftingError) as x:
            a.group_edit_begin([good] + make(G))                     # a valid record ahead of the bad one is not enqueued either
        assert x.value.rc == rc, what
        assert np.array_equal(a.digest(0, G), before), what
    ib = _sweep_inbox(G, F, workload.T0_MS + 2_000_000)
    harness.assert_outbox_equal(a.step(ib), b.step(ib), where="the step after the refusals")
    a.group_edit_begin([])                                            # n == 0: nothing to do


def test_per_group_restarts_in_a_live_node_through_group_edit_begin(tmp_path):
    """tests/test_group_edit_cpu.py's per-group restarts with every node an engine and the oracle in lock-step: the engine
    reopens through rafting_group_edit_begin, the oracle through the synchronous calls, and every step's outbox and the
    final states must be equal."""
    from tests.test_cluster_gpu import Pair
    from tests.test_group_edit_cpu import group_restarts

    class EditPair(Pair):
        def group_edit_begin(self, recs):
            self.e.group_edit_begin(recs)
            ep.apply_sync(self.o, recs)

    c = group_restarts(lambda cfg: EditPair(engine, cfg), 3, 41, tmp_path)
    for nd in c.nodes:
        for g in range(c.G):
            nd.sut.export(g)                                            # Pair.export insists on equal states


def test_group_edit_native_through_the_jni_glue(tmp_path):
    from tests import jni_exec
    from tests.jni_exec import Buf, buf_of_array, fn
    from tests.test_jni_glue_gpu import GlueEngine
    L = jni_exec.build(str(tmp_path))
    if L is None:
        pytest.skip("no gcc")
    G, R, rows, steps = 1024, 3, 4, 8
    cfg = abi.make_cfg(replicas=R, max_groups=G, max_rows=rows)
    o, e = binding.Oracle(cfg), GlueEngine(L, cfg, G, R - 1)
    init = harness.init_array(G, terms=np.arange(G) % 7)
    o.open_bulk(0, init), e.open_bulk(0, init)
    w1, w = workload.make_wl(11, 1, G, R - 1), workload.make_wl(11, rows, G, R - 1)
    harness.elect_all(o, w1), harness.elect_all(e, w1)
    edit = fn(L, "groupEditBegin", None, C.c_int64, C.POINTER(Buf), C.c_int32)
    prev, edited = None, np.zeros(0, np.int64)
    for k in range(steps):
        if k == 3:
            recs = np.array([edit_close(g) if g % 2 else
                             edit_open(g, runs=[(1, 1), (3, 2)], term=4, ballot=1, last_index=6, last_term=2, now_ms=workload.T0_MS)
                             for g in range(0, G, 7)], dtype=abi.GROUP_EDIT)
            L.fake_reset()
            edit(e.h, C.byref(buf_of_array(recs)), len(recs))
            assert L.fake_throws() == 0, L.fake_thrown_message()
            ep.apply_sync(o, recs)
            edited = recs["gid"].astype(np.int64)
        ib = workload.leader_inbox_host(w, k, prev)
        if k == 3 and ib.ev_meta is not None:                         # replies to RPCs planned before the edit are dropped
            ib.ev_meta[:, edited] = 0
        prev = o.step(ib)
        harness.assert_outbox_equal(prev, e.step(ib), where=f"step {k} through the natives")
    harness.assert_states_equal(o, e, range(G), R - 1, where="after the edits")
    bad = np.array([edit_open(G)], dtype=abi.GROUP_EDIT)
    L.fake_reset()
    edit(e.h, C.byref(buf_of_array(bad)), 1)
    assert L.fake_throws() == 1
    L.fake_reset()
    fn(L, "destroy", None, C.c_int64)(e.h)
