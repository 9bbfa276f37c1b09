"""Timers on the compact host path, on CPU: the due predicate, the pipelining rule and the compact encoding of sweep rows.

  * the predicate of rafting_timers_due_begin, restated in numpy over the oracle's exported state (tests/timers_model.py),
    selects exactly the groups that one oracle sweep step fires: on states of the config #3 / #5 streams and of cluster_sim
    runs, with closed groups, muted timers (a stale installSnapshot) and until == deadline
  * the pipelining rule: a cluster whose nodes step over the rule's lists (due list of the state d steps back, the lists in
    flight, the step's event gids) stays, tick after tick, in the state of the same cluster stepping the whole shard
  * a compact sweep step (compact.encode_inbox(sweep=True)) decodes to the dense inbox with row_now, through the compact model"""
import numpy as np
import pytest

from oracle import binding
from rafting_b200 import abi, compact, workload
from tests import compact_active_model as active
from tests import compact_model as model
from tests import harness
from tests import timers_model as tm
from tests.cluster_sim import Cluster
from tests.compact_model import EL, PT

U64 = np.uint64


def _stale_install(o, G, F, now, every=13):
    """A stale-term installSnapshot at every `every`-th follower: its election timer is left muted (Follower.java:134-137)."""
    ib = abi.Inbox(1, G, F, ent_cap=1)
    for g in range(0, G, every):
        s = o.export(g)
        if s.alive and s.role == abi.ROLE_FOLLOWER and s.current_term > 0:
            ib.is_request(0, g, now, leader=(s.current_term % (F + 1)), term=s.current_term - 1, last_included_index=0,
                          last_included_term=0, host_result=False)
    o.step(ib)


def _config3(k_steps, G=1024):
    def make():
        cfg, init, w = model._storm_open(G, 3, 4)
        o = binding.Oracle(cfg)
        o.open_bulk(0, init)
        prev = None
        for k in range(k_steps):
            prev = o.step(workload.vote_inbox_host(w, k, prev))
        _stale_install(o, G, 2, workload.T0_MS + 1000)
        for g in range(5, G, 97):
            o.close_group(g)
        return o, G, 2
    return make


def _config5(k_steps, G=1024):
    def make():
        cfg = abi.make_cfg(replicas=3, max_groups=G, max_rows=4, entry_pool_cap=4 * G * 50)
        o = binding.Oracle(cfg)
        o.open_bulk(0, harness.init_array(G, terms=np.arange(G) % 7))
        harness.elect_all(o, workload.make_wl(0x5EED0005, 1, G, 2))
        w = workload.make_wl(0x5EED0005, 4, G, 2)
        prev = None
        for k in range(k_steps):
            prev = o.step(workload.mixed_inbox_host(w, k, prev))
        for g in range(3, G, 61):
            o.close_group(g)
        return o, G, 2
    return make


def _cluster(ticks):
    def make():
        c = Cluster(lambda cfg: binding.Oracle(cfg), G=24, R=3, seed=5, drop_ppm=20_000)
        c.run(ticks // 2)
        c.cut = {c.leader_of(0)}
        c.run(ticks - ticks // 2)
        o = c.nodes[1].sut
        _stale_install(o, 24, 2, c.tick * 10 + 1_700_000_000_000, every=5)
        o.close_group(7)
        return o, 24, 2
    return make


SOURCES = {"config3": _config3(4), "config5": _config5(6), "cluster": _cluster(120)}


@pytest.mark.parametrize("source", sorted(SOURCES))
def test_due_predicate_is_what_one_oracle_sweep_fires(source):
    make = SOURCES[source]
    o, G, F = make()
    t0 = tm.table([o.export(g) for g in range(G)])
    armed = np.sort(t0["timer"][(t0["alive"] != 0) & (t0["timer"] > 0) & (t0["timer"] != tm.I64MAX)])
    assert len(armed) > 10
    assert (t0["alive"] == 0).any(), "closed groups"
    if source != "config5":
        assert ((t0["alive"] != 0) & (t0["timer"] == tm.I64MAX)).any(), "muted timers"
    for until in (int(armed[len(armed) // 2]), int(armed[len(armed) // 2]) - 1, int(armed[0]), int(armed[-1]) + 1):
        o, _, _ = make()                                                # a fresh oracle in the same state for every sweep
        before = [harness.state_bytes(o.export(g), F) for g in range(G)]
        want = tm.due(t0, until)
        assert (t0["timer"][want] == until).any() or until != int(armed[len(armed) // 2]), "until == a deadline"
        ib = abi.Inbox(1, G, F, with_ops=False, with_events=False, sweep=True)
        ib.row_now[0] = until
        o.step(ib)
        fired = np.array([harness.state_bytes(o.export(g), F) != before[g] for g in range(G)])
        assert np.array_equal(fired, want), f"until {until}: fired {np.flatnonzero(fired ^ want)[:10]} differ from the predicate"


@pytest.mark.parametrize("d", [0, 1, 3])
def test_pipelining_rule_keeps_a_cluster_in_the_whole_shard_sweep_state(d):
    G, R = 24, 3
    ref = Cluster(lambda cfg: binding.Oracle(cfg), G=G, R=R, seed=11, submit_ppm=40_000)
    pumps = []

    def make(cfg):
        p = tm.RulePump(binding.Oracle(cfg), G, R - 1, d)
        pumps.append(p)
        return p
    cand = Cluster(make, G=G, R=R, seed=11, submit_ppm=40_000)

    def tick(n, cut=None):
        for _ in range(n):
            if cut is not None:
                ref.cut = cand.cut = cut
            ref.step(); cand.step()
            for a, b in zip(ref.nodes, cand.nodes):
                for g in range(G):
                    assert harness.state_bytes(a.sut.export(g), R - 1) == harness.state_bytes(b.sut.export(g), R - 1), \
                        f"node {a.slot} group {g} at tick {ref.tick}"
    tick(100)
    victim = ref.leader_of(0)
    assert victim is not None
    tick(120, cut={victim})                                              # its followers lose their leader and elect
    tick(100, cut=set())
    ref.check(converged=False); cand.check(converged=False)
    listed = np.array([n for p in pumps for n in p.listed[1:]])
    assert listed.mean() < 0.8 * G, f"the lists hold {listed.mean():.1f} of {G} groups on average"
    assert sum(p.due_only for p in pumps) > 50                           # timers fired by the due list alone


@pytest.mark.parametrize("flags", [0, EL | PT])
@pytest.mark.parametrize("listed", [False, True])
def test_compact_sweep_step_decodes_to_the_dense_step_with_row_now(flags, listed):
    G, R, rows = 1024, 3, 4
    F = R - 1
    cfg = abi.make_cfg(replicas=R, max_groups=G, max_rows=rows, entry_pool_cap=rows * G * 50)
    o = binding.Oracle(cfg)
    o.open_bulk(0, harness.init_array(G, terms=np.arange(G) % 7))
    harness.elect_all(o, workload.make_wl(0x5EED0005, 1, G, F))
    w = workload.make_wl(0x5EED0005, rows, G, F)
    A = np.sort(np.random.default_rng(3).choice(G, 400, replace=False)).astype(np.uint32) if listed else None
    st, g_term = model.InFlight(G, F), np.array([o.export(g).current_term for g in range(G)], np.int64)
    prev, nxt, fired = None, None, 0
    for k in range(6):
        ib = workload.mixed_inbox_host(w, k, prev, gids=A)
        ib.row_now = np.zeros(rows, np.int64)
        base = int(ib.op_nr["x"][ib.op_meta != 0].min()) if (ib.op_meta != 0).any() else workload.T0_MS
        ib.row_now[k % 2] = base + 400 * k                                # a sweep in row 0 or row 1
        if k == 5:
            ib.op_meta = None; ib.ev_meta = None; ib.op_nr = ib.op_ab = ib.op_cd = ib.op_e = None; ib.ev_tn = ib.ev_el = None
        ci = compact.encode_inbox(ib, **(nxt or dict(tags=None, sent_term=None)), elections=bool(flags & EL), sweep=True)
        assert np.array_equal(ci.sweep, ib.row_now)
        if ci.reqs is not None:                                          # no record on a sweep row
            on = ci.sweep[ci.reqs.req["slot"] // ib.n] != 0
            assert not on.any()
            assert not (ci.sweep[ci.reqs.op_esc["slot"] // ib.n] != 0).any()
        if k == 5:
            assert ci.op_c is None and ci.ev_c is None and ci.reqs is None   # a sweep-only step
        dense = active.unpack(ci, g_term, st, flags, gids=A) if ci.op_c is not None or ci.ev_c is not None or ci.reqs is not None else None
        want = o.step(ib, threads=8)
        if dense is not None:                                            # the step reads what the dense step reads
            dense.row_now = ci.sweep
            sw = ib.row_now != 0
            if ib.op_meta is not None:
                keep = ~sw
                a_ops = ib.op_meta.copy(); a_ops[sw] = 0
                assert np.array_equal(a_ops[keep] & U64(0xFFFFFFFF), dense.op_meta[keep] & U64(0xFFFFFFFF))
            if ib.ev_meta is not None:
                assert np.array_equal(ib.ev_meta, dense.ev_meta)
        fired += int((want.plan_meta[ib.row_now != 0] != 0).sum()) + int((want.ballot_meta[ib.row_now != 0] != 0).sum())
        ep = np.zeros(G, abi.I64X2)
        for g in (range(G) if A is None else A.tolist()):
            s = o.export(g); ep[g] = (s.epoch_index, s.epoch_term)
        co = active.pack(want, ep, st, esc_cap=rows * G * F + 2 * rows * G, flags=flags, replies=ci.reqs is not None, gids=A)
        harness.assert_outbox_equal(want, compact.decode_outbox(co, elections=bool(flags & EL), prev_term=bool(flags & PT)),
                                    where=f"step {k}")
        g_term[np.arange(G) if A is None else A] = want.current_term[:ib.n]
        nxt, prev = model.next_of(want, co), want
    assert fired > 0


def test_encode_inbox_leaves_row_now_out_by_default():
    G, F, rows = 64, 2, 2
    ib = abi.Inbox(rows, G, F, sweep=True)
    ib.row_now[0] = workload.T0_MS
    ib.submit(1, 3, workload.T0_MS)
    ci = compact.encode_inbox(ib, None, None)
    assert getattr(ci, "sweep", None) is None
    cs = compact.encode_inbox(ib, None, None, sweep=True)
    assert np.array_equal(cs.sweep, ib.row_now) and np.array_equal(cs.op_c, ci.op_c)
