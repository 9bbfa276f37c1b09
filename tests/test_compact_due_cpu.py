"""Due steps on the compact host path, on CPU (rafting_step_begin_compact_due): the tail model against the oracle, a cluster of
nodes stepping over their event gids plus the tail, and the codec's padded inbox.

  * the tail (tests/due_model.py) over the oracle's exported state of the config #3 / #5 streams and of a cluster_sim run, with
    closed groups, muted timers (a stale installSnapshot) and until == a deadline; host lists that are empty, that hold due
    groups, and counts[3] below and above cap.  A sweep over host + tail leaves the shard as the whole-shard sweep does when
    counts[3] <= cap; above it, exactly the due groups past the tail are left untouched, and still due
  * a 3-node cluster_sim run of 320 ticks whose nodes step over their event gids plus the model's tail, with the cap following
    counts[3] d = 0, 1 and 3 steps behind, stays in the whole-shard cluster's state after every tick
  * compact.due_inbox: the host's positions encode as before, and the tail positions are empty"""
import numpy as np
import pytest

from oracle import binding
from rafting_b200 import abi, compact, workload
from tests import compact_model as model
from tests import due_model as dm
from tests import harness
from tests import timers_model as tm
from tests.cluster_sim import Cluster


def _stale_install(o, G, F, now, every):
    """a stale-term installSnapshot at every `every`-th follower leaves its election timer muted (Follower.java:134-137)"""
    ib = abi.Inbox(1, G, F, ent_cap=1)
    for g in range(0, G, every):
        s = o.export(g)
        if s.alive and s.role == abi.ROLE_FOLLOWER and s.current_term > 0:
            ib.is_request(0, g, now, leader=(s.current_term % (F + 1)), term=s.current_term - 1, last_included_index=0,
                          last_included_term=0, host_result=False)
    o.step(ib)


def _config3(G=1024):
    cfg, init, w = model._storm_open(G, 3, 4)
    o = binding.Oracle(cfg)
    o.open_bulk(0, init)
    prev = None
    for k in range(4):
        prev = o.step(workload.vote_inbox_host(w, k, prev))
    _stale_install(o, G, 2, workload.T0_MS + 1000, 13)
    for g in range(5, G, 97):
        o.close_group(g)
    return o, G, 2


def _config5(G=1024):
    cfg = abi.make_cfg(replicas=3, max_groups=G, max_rows=4, entry_pool_cap=4 * G * 50)
    o = binding.Oracle(cfg)
    o.open_bulk(0, harness.init_array(G, terms=np.arange(G) % 7))
    harness.elect_all(o, workload.make_wl(0x5EED0005, 1, G, 2))
    w = workload.make_wl(0x5EED0005, 4, G, 2)
    prev = None
    for k in range(6):
        prev = o.step(workload.mixed_inbox_host(w, k, prev))
    for g in range(3, G, 61):
        o.close_group(g)
    return o, G, 2


def _cluster():
    c = Cluster(lambda cfg: binding.Oracle(cfg), G=24, R=3, seed=5, drop_ppm=20_000)
    c.run(60)
    c.cut = {c.leader_of(0)}
    c.run(60)
    o = c.nodes[1].sut
    _stale_install(o, 24, 2, c.tick * 10 + 1_700_000_000_000, 5)
    o.close_group(7)
    return o, 24, 2


SOURCES = {"config3": _config3, "config5": _config5, "cluster": _cluster}


def _sweep(o, G, F, until, gids=None):
    """one sweep-only step at `until`, over the whole shard or the (sorted) list gids"""
    ib = abi.Inbox(1, G, F, with_ops=False, with_events=False, sweep=True)
    ib.row_now[0] = until
    o.step(ib if gids is None else tm.slice_inbox(ib, np.sort(gids)))


@pytest.mark.parametrize("source", sorted(SOURCES))
def test_tail_model_is_what_the_whole_shard_sweep_fires(source):
    make = SOURCES[source]
    o, G, F = make()
    t = tm.table([o.export(g) for g in range(G)])
    assert (t["alive"] == 0).any(), "closed groups"
    if source != "config5":
        assert ((t["alive"] != 0) & (t["timer"] == tm.I64MAX)).any(), "muted timers"
    armed = np.sort(t["timer"][(t["alive"] != 0) & (t["timer"] > 0) & (t["timer"] != tm.I64MAX)])
    until = int(armed[len(armed) // 2])                                   # a deadline: until == timer for some group
    due = np.flatnonzero(tm.due(t, until))
    assert (t["timer"][due] == until).any() and len(due) > 4
    rng = np.random.default_rng(1)
    cases = {                                                             # host list, cap
        "empty list, cap above": (np.zeros(0, np.int64), len(due) + 3),
        "list holding due groups": (np.sort(np.concatenate([due[::3], rng.choice(G, G // 8, replace=False)])), len(due)),
        "empty list, cap below": (np.zeros(0, np.int64), len(due) // 2),
        "list holding due groups, cap below": (np.unique(np.concatenate([due[1::4], np.arange(0, G, 11)])), 2),
    }
    for name, (host, cap) in cases.items():
        host = np.unique(host).astype(np.int64)
        tl, n_due = dm.tail(t, host, cap, until)
        want_due = np.setdiff1d(due, host)
        assert n_due == len(want_due), name
        k = min(n_due, cap)
        inc = lambda a: (np.diff(a.astype(np.int64)) > 0).all()
        assert len(tl) == cap and inc(tl[:k]) and inc(tl[k:]) and not np.isin(tl, host).any(), name
        assert np.array_equal(tl[:k], want_due[:k]) and not tm.due(t, until)[tl[k:]].any(), name
        assert ("below" in name) == (n_due > cap), name
        ref, _, _ = make()
        before = [harness.state_bytes(ref.export(g), F) for g in range(G)]
        _sweep(ref, G, F, until)
        cand, _, _ = make()
        _sweep(cand, G, F, until, gids=np.concatenate([host, tl.astype(np.int64)]))
        left = set(want_due[cap:].tolist())                               # due groups past the tail: untouched
        for g in range(G):
            got = harness.state_bytes(cand.export(g), F)
            want = before[g] if g in left else harness.state_bytes(ref.export(g), F)
            assert got == want, f"{name}: group {g}"
        if left:
            after = tm.table([cand.export(g) for g in range(G)])
            assert tm.due(after, until)[sorted(left)].all(), f"{name}: the groups left over stay due"


@pytest.mark.parametrize("d", [0, 1, 3])
def test_due_pump_keeps_a_cluster_in_the_whole_shard_sweep_state(d):
    G, R = 24, 3
    ref = Cluster(lambda cfg: binding.Oracle(cfg), G=G, R=R, seed=11, submit_ppm=40_000)
    pumps = []

    def make(cfg):
        p = dm.DuePump(binding.Oracle(cfg), G, R - 1, d, cap0=4)
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
    assert sum(p.overflows for p in pumps) == 0
    assert sum(sum(p.counts) for p in pumps) > 50                        # timers fired through the tail
    assert sum(p.fillers for p in pumps) > 0
    listed = np.array([n for p in pumps for n in p.listed[1:]])
    assert listed.mean() < 0.8 * G, f"the lists hold {listed.mean():.1f} of {G} groups on average"


def test_due_inbox_pads_the_tail_positions_empty():
    G, F, rows, cap = 256, 2, 3, 7
    w = workload.make_wl(0x5EED0005, rows, G, F)
    A = np.arange(3, G, 5, dtype=np.uint32)
    ib = workload.mixed_inbox_host(w, 1, None, gids=A)
    ib.row_now = np.zeros(rows, np.int64)
    ib.row_now[0] = workload.T0_MS + 300
    ib.op_meta[0] = 0
    ci = compact.encode_inbox(ib, None, None, sweep=True)
    di = compact.due_inbox(ib, cap)
    cd = compact.encode_inbox(di, None, None, sweep=True)
    n = len(A)
    assert cd.n == n + cap and np.array_equal(cd.gids, A) and np.array_equal(cd.sweep, ci.sweep)
    assert np.array_equal(cd.op_c[:, :n], ci.op_c) and not cd.op_c[:, n:].any()
    assert np.array_equal(cd.ev_c[:, :n], ci.ev_c) and not cd.ev_c[:, n:].any()
    if ci.reqs is not None:                                             # the request list: slot r * n + i becomes r * (n + cap) + i
        r, i = np.divmod(ci.reqs.req["slot"].astype(np.int64), n)
        assert np.array_equal(cd.reqs.req["slot"], r * (n + cap) + i)
    empty = compact.due_inbox(tm.slice_inbox(abi.Inbox(rows, G, F, sweep=True), np.zeros(0, np.uint32)), cap)
    assert empty.n == cap and len(empty.gids) == 0
