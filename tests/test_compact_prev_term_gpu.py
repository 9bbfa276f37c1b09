"""AE plans with an older prevLogTerm through the compact host path (`-m gpu`): config #3 and config #5 fed through
rafting_step_begin_compact_ex with RAFTING_COMPACT_PREV_TERM (alone and with RAFTING_COMPACT_ELECTIONS) must decode, step by
step, to the dense step of the oracle, and pack exactly what tests/compact_prev_term_model.py says: a twin engine runs the
same stream without the flag (whose pack the existing suites check against the older models), and the model turns its outbox
into the flagged one, which must equal the engine's plan_c and escape records bit for bit.  Flags change between steps, an
escape-list overflow falls back to the dense outbox, and kind-7 tags survive rafting_state_save / rafting_state_load."""
import numpy as np
import pytest

from oracle import binding
from rafting_b200 import abi, compact, ingest, workload
from tests import compact_prev_term_model as pt_model
from tests import harness
from tests.test_compact_prev_term_cpu import EL, PT, encode, next_of

pytestmark = pytest.mark.gpu


def _engines(G, R, rows, n, storm):
    """n engines and the oracle, opened alike: config #3 (a vote storm from followers) or config #5 (elected leaders)"""
    from rafting_b200 import engine
    if storm:
        cfg = abi.make_cfg(replicas=R, local_slot=1, max_groups=G, max_rows=rows, entry_pool_cap=workload.POOL_TERMS)
        init = harness.init_array(G, terms=1 + np.arange(G) % 5)
        init["last_index"] = 100 + np.arange(G) % 50
        init["last_term"] = 1 + np.arange(G) % 5
    else:
        cfg = abi.make_cfg(replicas=R, max_groups=G, max_rows=rows, entry_pool_cap=rows * G * 50)
        init = harness.init_array(G, terms=np.arange(G) % 7)
    es, o = [engine.Engine(cfg) for _ in range(n)], binding.Oracle(cfg)
    for s in es + [o]:
        s.open_bulk(0, init)
    if not storm:
        w1 = workload.make_wl(0x5EED0005, 1, G, R - 1)
        want = harness.elect_all(o, w1)
        for e in es:
            harness.assert_outbox_equal(want, harness.elect_all(e, w1), where="election (dense path)")
    return es, o


def _sorted_esc(co):
    esc = co.esc[:int(co.counts[0])].copy()
    return np.sort(esc, order=["kind", "slot"]).tobytes()


class Driver:
    """A pump around one engine under test (and, optionally, its unflagged twin), checked against the oracle every step."""

    def __init__(self, e, o, G, F, rows, twin=None):
        self.e, self.o, self.twin, self.G, self.F, self.rows = e, o, twin, G, F, rows
        self.nxt, self.prev = None, None
        self.ae = self.ae_words = self.kind7 = self.records = self.records0 = 0

    def step(self, ib, flags, esc_cap=None, where=""):
        rows, G, F = self.rows, self.G, self.F
        want = self.o.step(ib, threads=8)
        cap = rows * G * F + 2 * rows * G if esc_cap is None else esc_cap
        cin = encode(ib, self.nxt, flags)
        cout = compact.CompactOutbox(rows, G, F, esc_cap=cap)
        self.e.step_compact(cin, cout, reqs=cin.reqs, flags=flags)
        if self.twin is not None:
            cout0 = compact.CompactOutbox(rows, G, F, esc_cap=rows * G * F + 2 * rows * G)
            self.twin.step_compact(cin, cout0, reqs=cin.reqs, flags=flags & ~PT)
            model = pt_model.prev_term_words(cout0, cap) if flags & PT else cout0
            assert np.array_equal(cout.plan_c, model.plan_c), f"plan_c differs from the model, {where}"
            assert np.array_equal(cout.tags(), model.tags()) and np.array_equal(cout.tags(rpc_only=True), model.tags(rpc_only=True))
            assert np.array_equal(cout.counts, model.counts) and _sorted_esc(cout) == _sorted_esc(model), f"escape records, {where}"
            self.records0 += sum(int(r["kind"]) == abi.CESC_PLAN for r in cout0.esc[:int(cout0.counts[0])])
        if esc_cap is None:
            harness.assert_outbox_equal(want, compact.decode_outbox(cout, elections=bool(flags & EL), prev_term=bool(flags & PT)),
                                        where=where)
            k = cout.plan_c & np.uint32(7)
            esc = ((cout.plan_c >> np.uint32(4)) & np.uint32(1)) != 0
            self.ae += int(((want.plan_meta & np.uint64(0xF)) == abi.PLAN_AE).sum())
            self.ae_words += int((((k == abi.PLAN_AE) & ~esc) | (k == abi.CPLAN_AE_PREV_TERM)).sum())
            self.kind7 += int((k == abi.CPLAN_AE_PREV_TERM).sum())
            self.records += sum(int(r["kind"]) == abi.CESC_PLAN for r in cout.esc[:int(cout.counts[0])])
        self.nxt, self.prev = next_of(want, cout, flags), want
        return cin, want, cout


def _run(G, R, rows, steps, flags, storm):
    (e, e0), o = _engines(G, R, rows, 2, storm)
    F = R - 1
    d = Driver(e, o, G, F, rows, twin=e0)
    w = workload.make_wl(0x5EED0003 if storm else 0x5EED0005, rows, G, F, **(dict(local_slot=1) if storm else {}))
    for k in range(steps):
        ib = workload.vote_inbox_host(w, k, d.prev) if storm else workload.mixed_inbox_host(w, k, d.prev)
        d.step(ib, flags, where=f"flags {flags}, step {k}")
    harness.assert_states_equal(o, e, list(range(0, G, max(1, G // 97))) + [G - 1], F, where=f"flags {flags} end")
    return d


@pytest.mark.parametrize("flags", [PT, EL | PT])
def test_config3_class_sorted_launch(flags):
    d = _run(G=16384, R=5, rows=1, steps=16, flags=flags, storm=True)
    assert d.kind7 > 1000 and d.records <= 0.1 * d.records0, vars(d)
    if flags == EL | PT:
        assert d.ae_words >= 0.95 * d.ae, vars(d)


@pytest.mark.parametrize("flags", [PT, EL | PT])
def test_config3_unsorted_launch(flags):
    d = _run(G=1024, R=5, rows=1, steps=16, flags=flags, storm=True)
    assert d.kind7 > 100 and d.records < d.records0, vars(d)


@pytest.mark.parametrize("flags", [PT, EL | PT])
def test_config5_four_rows(flags):
    d = _run(G=16384, R=3, rows=4, steps=24, flags=flags, storm=False)
    assert d.kind7 > 1000 and d.records <= 0.5 * d.records0, vars(d)


def test_flags_change_between_steps():
    G, R, rows = 2048, 5, 1
    F = R - 1
    (e,), o = _engines(G, R, rows, 1, storm=True)
    d = Driver(e, o, G, F, rows)
    w = workload.make_wl(0x5EED0003, rows, G, F, local_slot=1)
    seq = [PT, 0, EL | PT, EL, PT, EL | PT, 0, EL | PT, PT, EL]
    for k in range(20):
        flags = seq[k % len(seq)]
        d.step(workload.vote_inbox_host(w, k, d.prev), flags, where=f"step {k} flags {flags}")
    assert d.kind7 > 0
    harness.assert_states_equal(o, e, list(range(0, G, 31)) + [G - 1], F, where="changing flags end")


def test_escape_overflow_falls_back_to_the_dense_outbox():
    G, R, rows = 1024, 3, 4
    F = R - 1
    (e,), o = _engines(G, R, rows, 1, storm=False)
    d = Driver(e, o, G, F, rows)
    w = workload.make_wl(0x5EED0005, rows, G, F)
    for k in range(10):
        d.step(workload.mixed_inbox_host(w, k, d.prev), EL | PT, where=f"step {k}")
    _, want, cout = d.step(workload.mixed_inbox_host(w, 10, d.prev), EL | PT, esc_cap=4)
    assert int(cout.counts[0]) > 4
    with pytest.raises(OverflowError):
        compact.decode_outbox(cout, elections=True, prev_term=True)
    with pytest.raises(OverflowError):
        ingest.Dispatch(G, F, 0).crequests(cout, rows, EL | PT)
    dense = abi.Outbox(rows, G, F, G)
    e.step_fetch_dense(0, dense.as_c())
    harness.assert_outbox_equal(want, dense, where="dense fallback")
    for k in range(11, 16):                                                    # the stream goes on compact
        d.step(workload.mixed_inbox_host(w, k, d.prev), EL | PT, where=f"after the fallback, step {k}")
    harness.assert_states_equal(o, e, list(range(0, G, 31)) + [G - 1], F, where="after the fallback")


def test_kind7_tags_survive_state_save_and_load(tmp_path):
    from rafting_b200 import engine
    G, R, rows = 2048, 3, 4
    F = R - 1
    (e,), o = _engines(G, R, rows, 1, storm=False)
    d = Driver(e, o, G, F, rows)
    w = workload.make_wl(0x5EED0005, rows, G, F)
    k = 0
    while True:
        _, _, cout = d.step(workload.mixed_inbox_host(w, k, d.prev), PT, where=f"before the save, step {k}")
        k += 1
        held = ((cout.plan_c & np.uint32(7)) == abi.CPLAN_AE_PREV_TERM) & (cout.tags() < 32)
        if held.any() or k == 30:
            break
    assert held.any(), "no kind-7 plan took a tag before the save"
    path = str(tmp_path / "shard.img")
    e.state_save(path)
    e2 = engine.Engine(e.cfg)
    e2.state_load(path)
    d.e = e2
    for k in range(k, k + 12):                                                 # the acks to those plans come back compact
        d.step(workload.mixed_inbox_host(w, k, d.prev), PT, where=f"after the load, step {k}")
    harness.assert_states_equal(o, e2, list(range(0, G, 31)) + [G - 1], F, where="after the load")


def test_flags_4_and_5_are_accepted_and_unknown_bits_refused():
    from rafting_b200 import engine
    (e,), _ = _engines(64, 3, 1, 1, storm=True)
    w = workload.make_wl(0x5EED0003, 1, 64, 2, local_slot=1)
    ib = workload.vote_inbox_host(w, 0, None)
    for flags in (PT, EL | PT):
        cin = encode(ib, None, flags)
        e.step_compact(cin, compact.CompactOutbox(1, 64, 2), reqs=cin.reqs, flags=flags)
    for flags in (2, 8, PT | 8, 0x80000000):
        cin = encode(ib, None, 0)
        with pytest.raises(engine.RaftingError) as ex:
            e.step_compact(cin, compact.CompactOutbox(1, 64, 2), reqs=cin.reqs, flags=flags)
        assert ex.value.rc == -1, flags
