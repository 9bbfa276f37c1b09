"""Elections through the compact host path (`-m gpu`): a config #3 vote storm fed through rafting_step_begin_compact_ex with
RAFTING_COMPACT_ELECTIONS (ballots as plan_c lanes, vote replies as ev_c words, vote requests as records) must be, once
decoded, bit for bit the dense step of the oracle on the same logical stream, in the class-sorted launch (G >= 2048) and the
unsorted one.  Flagged and unflagged steps mix freely, an escape-list overflow falls back losslessly to the dense outbox, and
the tags ballots hold survive rafting_state_save / rafting_state_load."""
import numpy as np
import pytest

from oracle import binding
from rafting_b200 import abi, compact, workload
from tests import harness
from tests.test_compact_elections_cpu import Ratios, _encode, _flagged_next

pytestmark = pytest.mark.gpu
U64 = np.uint64
EL = abi.COMPACT_ELECTIONS


def _storm_pair(G, R, rows):
    from rafting_b200 import engine
    cfg = abi.make_cfg(replicas=R, local_slot=1, max_groups=G, max_rows=rows, entry_pool_cap=workload.POOL_TERMS)
    e, o = engine.Engine(cfg), binding.Oracle(cfg)
    init = harness.init_array(G, terms=1 + np.arange(G) % 5)
    init["last_index"] = 100 + np.arange(G) % 50
    init["last_term"] = 1 + np.arange(G) % 5
    e.open_bulk(0, init), o.open_bulk(0, init)
    return e, o, workload.make_wl(0x5EED0003, rows, G, R - 1, local_slot=1)


class Driver:
    """Keeps the host-side bookkeeping of a pump: what the next step's encoder needs from the last one, flagged or not."""

    def __init__(self, e, o, G, F, rows):
        self.e, self.o, self.G, self.F, self.rows = e, o, G, F, rows
        self.nxt, self.prev0, self.prev = None, (None, None, None), None

    def step(self, ib, flagged: bool, esc_cap=None, where=""):
        rows, G, F = self.rows, self.G, self.F
        want = self.o.step(ib, threads=8)
        cap = rows * G * F + 2 * rows * G if esc_cap is None else esc_cap
        cout = compact.CompactOutbox(rows, G, F, esc_cap=cap)
        if flagged:
            cin = _encode(ib, self.nxt)
            self.e.step_compact(cin, cout, reqs=cin.reqs, flags=EL)
        else:
            cin = compact.encode_inbox(ib, *self.prev0)
            self.e.step_compact(cin, cout, reqs=cin.reqs if cin.reqs is not None else compact.CompactRequests())
        if esc_cap is None:
            harness.assert_outbox_equal(want, compact.decode_outbox(cout, elections=flagged), where=where)
        self.nxt = _flagged_next(want, cout) if flagged else dict(
            tags=cout.tags(rpc_only=True), sent_term=cout.current_term.copy(), sent_inc=cout.incarnation.copy(),
            ballot_term=np.zeros((rows, G), np.int64), ballot_inc=np.zeros((rows, G), U64),
            ballot_tags=np.full((rows, G, F), abi.CTAG_NONE, np.uint8))                     # escaped ballots: no tags
        self.prev0 = (cout.tags(), cout.current_term.copy(), cout.incarnation.copy())
        self.prev = want
        return cin, want, cout


def _run_storm(G, R, rows, steps, settle=2):
    e, o, w = _storm_pair(G, R, rows)
    d = Driver(e, o, G, R - 1, rows)
    ratios = Ratios()
    for k in range(steps):
        ib = workload.vote_inbox_host(w, k, d.prev)
        cin, want, cout = d.step(ib, True, where=f"flagged storm step {k}")
        if k >= settle:
            ratios.add(ib, cin, want, cout)
    harness.assert_states_equal(o, e, list(range(0, G, max(1, G // 97))) + [G - 1], R - 1, where="flagged storm end")
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
    from tests.test_compact_requests_gpu import _pair
    G, R, rows, steps, settle = 16384, 3, 4, 32, 8
    F = R - 1
    e, o = _pair(G, R, rows)
    d = Driver(e, o, G, F, rows)
    w = workload.make_wl(0x5EED0005, rows, G, F)
    flagged = Ratios()
    for k in range(steps):
        ib = workload.mixed_inbox_host(w, k, d.prev)
        plain = compact.encode_inbox(ib, *d.prev0)                            # what the unflagged encoder would send
        cin, want, cout = d.step(ib, True, where=f"flagged config #5 step {k}")
        if k >= settle:
            flagged.add(ib, cin, want, cout)
            plain_records = 0 if plain.reqs is None else len(plain.reqs.req)
            flagged_ae = 0 if cin.reqs is None else int((((cin.reqs.req["meta"] >> np.uint32(11)) & np.uint32(3)) == 0).sum())
            assert flagged_ae == plain_records, k
    harness.assert_states_equal(o, e, list(range(0, G, 97)) + [G - 1], F, where="flagged config #5 end")
    assert flagged.ae_records >= 0.9 * flagged.ae > 0, vars(flagged)


@pytest.mark.parametrize("first_flagged", [True, False])
def test_flagged_and_unflagged_steps_mix_exactly(first_flagged):
    G, R, rows = 2048, 5, 1
    e, o, w = _storm_pair(G, R, rows)
    d = Driver(e, o, G, R - 1, rows)
    for k in range(24):
        flagged = (k // 3) % 2 == (0 if first_flagged else 1)                  # three steps each way, alternating
        d.step(workload.vote_inbox_host(w, k, d.prev), flagged, where=f"step {k} flagged={flagged}")
    harness.assert_states_equal(o, e, list(range(0, G, 31)) + [G - 1], R - 1, where="mixed flags end")


def test_escape_overflow_with_elections_falls_back_to_the_dense_outbox():
    G, R, rows = 1024, 5, 1
    F = R - 1
    e, o, w = _storm_pair(G, R, rows)
    d = Driver(e, o, G, F, rows)
    for k in range(4):
        d.step(workload.vote_inbox_host(w, k, d.prev), True, where=f"step {k}")
    ib = workload.vote_inbox_host(w, 4, d.prev)
    _, want, cout = d.step(ib, True, esc_cap=4)
    assert int(cout.counts[0]) > 4
    with pytest.raises(OverflowError):
        compact.decode_outbox(cout, elections=True)
    dense = abi.Outbox(rows, G, F, G)
    e.step_fetch_dense(0, dense.as_c())
    harness.assert_outbox_equal(want, dense, where="dense fallback")
    # the overflowed step's compact columns are still right, so the stream goes on compact
    for k in range(5, 9):
        d.step(workload.vote_inbox_host(w, k, d.prev), True, where=f"after the fallback, step {k}")


def test_ballot_tags_survive_state_save_and_load(tmp_path):
    from rafting_b200 import engine
    G, R, rows = 2048, 5, 1
    F = R - 1
    e, o, w = _storm_pair(G, R, rows)
    d = Driver(e, o, G, F, rows)
    for k in range(6):
        d.step(workload.vote_inbox_host(w, k, d.prev), True, where=f"before the save, step {k}")
    assert (d.nxt["ballot_tags"] != abi.CTAG_NONE).any()                              # ballots of the last step hold tags
    path = str(tmp_path / "shard.img")
    e.state_save(path)
    e2 = engine.Engine(e.cfg)
    e2.state_load(path)
    d.e = e2
    ratios = Ratios()
    for k in range(6, 30):
        ib = workload.vote_inbox_host(w, k, d.prev)
        cin, want, cout = d.step(ib, True, where=f"after the load, step {k}")
        ratios.add(ib, cin, want, cout)
    ratios.assert_mostly_compact()
    harness.assert_states_equal(o, e2, list(range(0, G, 31)) + [G - 1], F, where="after the load")


def test_vote_records_without_the_flag_are_malformed():
    G, R, rows = 1024, 5, 1
    F = R - 1
    e, o, w = _storm_pair(G, R, rows)
    d = Driver(e, o, G, F, rows)
    for k in range(3):
        d.step(workload.vote_inbox_host(w, k, d.prev), True, where=f"step {k}")
    ib = workload.vote_inbox_host(w, 3, d.prev)
    cin = _encode(ib, d.nxt)
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
    want = o.step(want_ib)
    cout = compact.CompactOutbox(rows, G, F, esc_cap=rows * G * F + 2 * rows * G)
    e.step_compact(cin, cout, reqs=cin.reqs)
    got = compact.decode_outbox(cout)
    harness.assert_outbox_equal(want, got, where="vote records without the flag")
    for s in cin.reqs.req["slot"][vk != 0]:
        assert (int(got.rep_meta.reshape(-1)[int(s)]) >> 8) == abi.ERR["BAD_EVENT"]


def test_unknown_flags_are_refused():
    from rafting_b200 import engine
    e, _, w = _storm_pair(64, 3, 1)
    cin = compact.encode_inbox(workload.vote_inbox_host(w, 0, None), None, None, None)
    with pytest.raises(engine.RaftingError) as ex:
        e.step_compact(cin, compact.CompactOutbox(1, 64, 2), reqs=cin.reqs, flags=2)
    assert ex.value.rc == -1
