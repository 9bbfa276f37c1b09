"""AE plans with an older prevLogTerm through the compact host path (`-m gpu`): config #3 and config #5 fed through
rafting_step_begin_compact_ex with RAFTING_COMPACT_PREV_TERM (alone and with RAFTING_COMPACT_ELECTIONS) must decode, step by
step, to the dense step of the oracle, and pack exactly what tests/compact_model.py says: a twin engine runs the
same stream without the flag (whose pack the other compact suites check against the model), and the model's prev_term_words
turns its outbox into the flagged one, which must equal the engine's plan_c and escape records bit for bit.  Flags change between steps, an
escape-list overflow falls back to the dense outbox, and kind-7 tags survive rafting_state_save / rafting_state_load."""
import numpy as np
import pytest

from rafting_b200 import abi, compact, ingest, workload
from tests import harness
from tests.compact_model import EL, PT, Driver, encode

pytestmark = pytest.mark.gpu


def _run(G, R, rows, steps, flags, storm):
    d = Driver(G, R, rows, storm, twin=True)
    for k in range(steps):
        d.step(d.inbox(k), flags, empty_list=True, where=f"flags {flags}, step {k}")
    harness.assert_states_equal(d.o, d.e, list(range(0, G, max(1, G // 97))) + [G - 1], R - 1, where=f"flags {flags} end")
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
    d = Driver(G, R, rows, storm=True)
    seq = [PT, 0, EL | PT, EL, PT, EL | PT, 0, EL | PT, PT, EL]
    for k in range(20):
        flags = seq[k % len(seq)]
        d.step(d.inbox(k), flags, empty_list=True, where=f"step {k} flags {flags}")
    assert d.kind7 > 0
    harness.assert_states_equal(d.o, d.e, list(range(0, G, 31)) + [G - 1], F, where="changing flags end")


def test_escape_overflow_falls_back_to_the_dense_outbox():
    G, R, rows = 1024, 3, 4
    F = R - 1
    d = Driver(G, R, rows, storm=False)
    for k in range(10):
        d.step(d.inbox(k), EL | PT, empty_list=True, where=f"step {k}")
    _, want, cout = d.step(d.inbox(10), EL | PT, empty_list=True, esc_cap=4)
    assert int(cout.counts[0]) > 4
    with pytest.raises(OverflowError):
        compact.decode_outbox(cout, elections=True, prev_term=True)
    with pytest.raises(OverflowError):
        ingest.Dispatch(G, F, 0).crequests(cout, rows, EL | PT)
    dense = abi.Outbox(rows, G, F, G)
    d.e.step_fetch_dense(0, dense.as_c())
    harness.assert_outbox_equal(want, dense, where="dense fallback")
    for k in range(11, 16):                                                    # the stream goes on compact
        d.step(d.inbox(k), EL | PT, empty_list=True, where=f"after the fallback, step {k}")
    harness.assert_states_equal(d.o, d.e, list(range(0, G, 31)) + [G - 1], F, where="after the fallback")


def test_kind7_tags_survive_state_save_and_load(tmp_path):
    from rafting_b200 import engine
    G, R, rows = 2048, 3, 4
    F = R - 1
    d = Driver(G, R, rows, storm=False)
    k = 0
    while True:
        _, _, cout = d.step(d.inbox(k), PT, empty_list=True, where=f"before the save, step {k}")
        k += 1
        held = ((cout.plan_c & np.uint32(7)) == abi.CPLAN_AE_PREV_TERM) & (cout.tags() < 32)
        if held.any() or k == 30:
            break
    assert held.any(), "no kind-7 plan took a tag before the save"
    path = str(tmp_path / "shard.img")
    d.e.state_save(path)
    e2 = engine.Engine(d.e.cfg)
    e2.state_load(path)
    d.e = e2
    for k in range(k, k + 12):                                                 # the acks to those plans come back compact
        d.step(d.inbox(k), PT, empty_list=True, where=f"after the load, step {k}")
    harness.assert_states_equal(d.o, e2, list(range(0, G, 31)) + [G - 1], F, where="after the load")


def test_flags_4_and_5_are_accepted_and_unknown_bits_refused():
    from rafting_b200 import engine
    d = Driver(64, 3, 1, storm=True)
    ib = workload.vote_inbox_host(d.w, 0, None)
    for flags in (PT, EL | PT):
        cin = encode(ib, None, flags, empty_list=True)
        d.e.step_compact(cin, compact.CompactOutbox(1, 64, 2), reqs=cin.reqs, flags=flags)
    for flags in (2, 8, PT | 8, 0x80000000):
        cin = encode(ib, None, 0, empty_list=True)
        with pytest.raises(engine.RaftingError) as ex:
            d.e.step_compact(cin, compact.CompactOutbox(1, 64, 2), reqs=cin.reqs, flags=flags)
        assert ex.value.rc == -1, flags
