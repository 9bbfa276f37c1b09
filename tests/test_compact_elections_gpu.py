"""Elections through the compact host path (`-m gpu`): a config #3 vote storm fed through rafting_step_begin_compact_ex with
RAFTING_COMPACT_ELECTIONS (ballots as plan_c lanes, vote replies as ev_c words, vote requests as records) must be, once
decoded, bit for bit the dense step of the oracle on the same logical stream, in the class-sorted launch (G >= 2048) and the
unsorted one.  Flagged and unflagged steps mix freely, an escape-list overflow falls back losslessly to the dense outbox, and
the tags ballots hold survive rafting_state_save / rafting_state_load."""
import numpy as np
import pytest

from rafting_b200 import abi, compact, workload
from tests import harness
from tests.compact_model import EL, Driver, Ratios, encode

pytestmark = pytest.mark.gpu


def _run_storm(G, R, rows, steps, settle=2):
    d = Driver(G, R, rows, storm=True)
    ratios = Ratios()
    for k in range(steps):
        ib = d.inbox(k)
        cin, want, cout = d.step(ib, EL, empty_list=False, where=f"flagged storm step {k}")
        if k >= settle:
            ratios.add(ib, cin, want, cout)
    harness.assert_states_equal(d.o, d.e, list(range(0, G, max(1, G // 97))) + [G - 1], R - 1, where="flagged storm end")
    return ratios


def test_config3_with_compact_elections_class_sorted_launch():
    _run_storm(G=16384, R=5, rows=1, steps=24).assert_mostly_compact()


def test_config3_with_compact_elections_unsorted_launch():
    _run_storm(G=1024, R=5, rows=1, steps=24).assert_mostly_compact()


def test_config3_with_compact_elections_three_replicas():
    _run_storm(G=4096, R=3, rows=1, steps=24).assert_mostly_compact()


def test_config3_with_compact_elections_two_rows_stays_exact():
    r = _run_storm(G=2048, R=5, rows=2, steps=24)
    assert r.ballot_lanes > 0 and r.reply_words > 0


def test_config5_with_the_flag_keeps_its_appendentries_compact():
    G, R, rows, steps, settle = 16384, 3, 4, 32, 8
    F = R - 1
    d = Driver(G, R, rows, storm=False)
    flagged = Ratios()
    for k in range(steps):
        ib = d.inbox(k)
        plain = encode(ib, d.nxt, 0, empty_list=False)                        # what the unflagged encoder would send
        cin, want, cout = d.step(ib, EL, empty_list=False, where=f"flagged config #5 step {k}")
        if k >= settle:
            flagged.add(ib, cin, want, cout)
            plain_records = 0 if plain.reqs is None else len(plain.reqs.req)
            flagged_ae = 0 if cin.reqs is None else int((((cin.reqs.req["meta"] >> np.uint32(11)) & np.uint32(3)) == 0).sum())
            assert flagged_ae == plain_records, k
    harness.assert_states_equal(d.o, d.e, list(range(0, G, 97)) + [G - 1], F, where="flagged config #5 end")
    assert flagged.ae_records >= 0.9 * flagged.ae > 0, vars(flagged)


@pytest.mark.parametrize("first_flagged", [True, False])
def test_flagged_and_unflagged_steps_mix_exactly(first_flagged):
    G, R, rows = 2048, 5, 1
    d = Driver(G, R, rows, storm=True)
    for k in range(24):
        flagged = (k // 3) % 2 == (0 if first_flagged else 1)                  # three steps each way, alternating
        d.step(d.inbox(k), EL if flagged else 0, empty_list=not flagged, where=f"step {k} flagged={flagged}")
    harness.assert_states_equal(d.o, d.e, list(range(0, G, 31)) + [G - 1], R - 1, where="mixed flags end")


def test_escape_overflow_with_elections_falls_back_to_the_dense_outbox():
    G, R, rows = 1024, 5, 1
    F = R - 1
    d = Driver(G, R, rows, storm=True)
    for k in range(4):
        d.step(d.inbox(k), EL, empty_list=False, where=f"step {k}")
    _, want, cout = d.step(d.inbox(4), EL, empty_list=False, esc_cap=4)
    assert int(cout.counts[0]) > 4
    with pytest.raises(OverflowError):
        compact.decode_outbox(cout, elections=True)
    dense = abi.Outbox(rows, G, F, G)
    d.e.step_fetch_dense(0, dense.as_c())
    harness.assert_outbox_equal(want, dense, where="dense fallback")
    # the overflowed step's compact columns are still right, so the stream goes on compact
    for k in range(5, 9):
        d.step(d.inbox(k), EL, empty_list=False, where=f"after the fallback, step {k}")


def test_ballot_tags_survive_state_save_and_load(tmp_path):
    from rafting_b200 import engine
    G, R, rows = 2048, 5, 1
    F = R - 1
    d = Driver(G, R, rows, storm=True)
    for k in range(6):
        d.step(d.inbox(k), EL, empty_list=False, where=f"before the save, step {k}")
    assert (d.nxt["ballot_tags"] != abi.CTAG_NONE).any()                              # ballots of the last step hold tags
    path = str(tmp_path / "shard.img")
    d.e.state_save(path)
    e2 = engine.Engine(d.e.cfg)
    e2.state_load(path)
    d.e = e2
    ratios = Ratios()
    for k in range(6, 30):
        ib = d.inbox(k)
        cin, want, cout = d.step(ib, EL, empty_list=False, where=f"after the load, step {k}")
        ratios.add(ib, cin, want, cout)
    ratios.assert_mostly_compact()
    harness.assert_states_equal(d.o, e2, list(range(0, G, 31)) + [G - 1], F, where="after the load")


def test_vote_records_without_the_flag_are_malformed():
    G, R, rows = 1024, 5, 1
    F = R - 1
    d = Driver(G, R, rows, storm=True)
    for k in range(3):
        d.step(d.inbox(k), EL, empty_list=False, where=f"step {k}")
    ib = d.inbox(3)
    cin = encode(ib, d.nxt, EL, empty_list=False)
    vk = (cin.reqs.req["meta"] >> np.uint32(11)) & np.uint32(3)
    assert (vk != 0).any()
    # without the flag the same records are answered with BAD_EVENT, exactly as the oracle answers malformed ops there
    want_ib = ib
    for s in cin.reqs.req["slot"][vk != 0]:
        r, i = divmod(int(s), G)
        want_ib.op_meta[r, i] = abi.COP_MALFORMED
        want_ib.op_nr[r, i] = (cin.row_base[r], 0); want_ib.op_ab[r, i] = (0, 0); want_ib.op_cd[r, i] = (0, 0); want_ib.op_e[r, i] = 0
    want_ib.ev_meta[...] = 0                                                    # and no events: the words mean nothing unflagged
    cin.ev_c = None; cin.esc = np.zeros(0, dtype=abi.CESC_IN)
    want = d.o.step(want_ib)
    cout = compact.CompactOutbox(rows, G, F, esc_cap=rows * G * F + 2 * rows * G)
    d.e.step_compact(cin, cout, reqs=cin.reqs)
    got = compact.decode_outbox(cout)
    harness.assert_outbox_equal(want, got, where="vote records without the flag")
    for s in cin.reqs.req["slot"][vk != 0]:
        assert (int(got.rep_meta.reshape(-1)[int(s)]) >> 8) == abi.ERR["BAD_EVENT"]


def test_unknown_flags_are_refused():
    from rafting_b200 import engine
    d = Driver(64, 3, 1, storm=True)
    cin = compact.encode_inbox(workload.vote_inbox_host(d.w, 0, None), None, None, None)
    with pytest.raises(engine.RaftingError) as ex:
        d.e.step_compact(cin, compact.CompactOutbox(1, 64, 2), reqs=cin.reqs, flags=2)
    assert ex.value.rc == -1
