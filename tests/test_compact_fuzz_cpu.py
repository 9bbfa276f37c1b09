"""The compact fuzz matrix (tests/compact_model.COMPACT_FUZZ) without a GPU: every case's stream through the codec and the
kernel model around the oracle, at a reduced step count, with the coverage each case is there for; the matrix reaches every
step kernel and launch mode the compact path can take; a model that loses one escape record is caught; and the codec's
fixes, each on the smallest inbox that shows it."""
import numpy as np
import pytest

from oracle import binding
from rafting_b200 import abi, compact
from tests import compact_model as model
from tests import harness, launch_model
from tests.compact_model import COMPACT_FUZZ, EL, PT

U64 = np.uint64


def compact_reachable() -> set:
    """Every (kernels, mode) a compact step can take: R = 2..17 (F <= 16: op_unavail is a 16-bit mask), both sides of the sort
    threshold, with and without a request list."""
    return {launch_model.kernels(R, n, fl) for R in range(2, 18) for n in (launch_model.SORT_MIN_N - 1, launch_model.SORT_MIN_N)
            for fl in (0, abi.INBOX_NO_REQUESTS)}


def test_matrix_reaches_every_compact_launch():
    covered = set()
    for case in COMPACT_FUZZ:
        assert case.R <= 17 and case.tail == 0, case.id
        covered.add(launch_model.kernels(case.R, case.n))
    missing = compact_reachable() - covered
    assert not missing, missing
    assert {c.entry for c in COMPACT_FUZZ} == {"whole", "active", "sweep", "active-sweep", "due"}
    assert {c.cflags for c in COMPACT_FUZZ} == {0, EL, PT, EL | PT}
    assert any(c.cfg_flags == model.CFG_BOTH for c in COMPACT_FUZZ)
    assert 0.35 <= np.mean([c.wide for c in COMPACT_FUZZ]) <= 0.65


_COVERAGE = {}


def coverage(case) -> model.StreamCoverage:
    """The case's run through the model at cpu_steps, once per session (the matrix-wide check reuses it)."""
    if case.id not in _COVERAGE:
        _COVERAGE[case.id] = model.FuzzPump(case).run(case.cpu_steps)
    return _COVERAGE[case.id]


@pytest.mark.parametrize("case", [pytest.param(c, id=c.id) for c in COMPACT_FUZZ])
def test_compact_fuzz_case_on_the_model(case):
    """The case through encode -> model unpack and oracle -> model pack -> decode, checked every step; then the stream went
    where the case is for."""
    cov = coverage(case)
    assert launch_model.kernels(case.R, case.n) in cov.launches or case.entry == "due", cov.launches
    assert cov.roles == {0, 1, 2}, cov.roles
    assert len(cov.errs) > 3, cov.errs
    acks = {abi.EV_AE_ACK}
    assert acks <= cov.words and acks <= cov.escaped, (cov.words, cov.escaped)
    if case.cflags & EL:
        assert {abi.EV_PV_REPLY, abi.EV_RV_REPLY} & cov.words, cov.words
        assert cov.ballot_lanes > 0
    assert {abi.EV_PV_REPLY, abi.EV_RV_REPLY} <= cov.escaped, cov.escaped
    if case.cflags & PT:
        assert cov.kind7 > 0
    if case.wide:
        assert cov.far > 0 and cov.wide_records >= 10, (cov.far, cov.wide_records)
    assert cov.overflows == 1
    if case.entry == "due":
        assert cov.due_over and cov.due_under, (cov.due_over, cov.due_under)


def test_every_event_kind_travels_both_ways():
    """Over the matrix, IS acks as words and as records too."""
    words, escaped = set(), set()
    for case in COMPACT_FUZZ:
        cov = coverage(case)
        words |= cov.words; escaped |= cov.escaped
    kinds = {abi.EV_AE_ACK, abi.EV_IS_ACK, abi.EV_PV_REPLY, abi.EV_RV_REPLY}
    assert kinds <= words and kinds <= escaped, (words, escaped)


class _DropsOneEscape(model.FuzzPump):
    """A kernel model whose pack loses one escape record."""

    def _pack(self, want, L, cap, replies):
        co = super()._pack(want, L, cap, replies)
        n = int(co.counts[0])
        if 0 < n <= co.esc_cap:
            co.esc[n // 2:n - 1] = co.esc[n // 2 + 1:n].copy()
            co.counts[0] = n - 1
        return co


def test_a_model_that_drops_an_escape_record_is_caught():
    case = COMPACT_FUZZ[0]
    with pytest.raises(AssertionError, match="pack -> decode"):
        _DropsOneEscape(case).run(2)


def _one_group(rows=1, F=2):
    cfg = abi.make_cfg(replicas=F + 1, max_groups=1, max_rows=rows, entry_pool_cap=16)
    o = binding.Oracle(cfg)
    o.open_bulk(0, harness.init_array(1, terms=[3]))
    return o, abi.Inbox(rows, 1, F, ent_cap=4)


def test_requests_of_a_no_requests_step_travel_as_refused_ops():
    """A step flagged INBOX_NO_REQUESTS that holds an AppendEntries anyway: the dense step answers it BAD_EVENT and does
    nothing else.  The encoder used to put it in the request list, so the compact step would have applied it."""
    o, ib = _one_group()
    ib.ae_request(0, 0, harness.T0, 1, 3, 0, 0, [3])
    ib.flags |= abi.INBOX_NO_REQUESTS
    ci = compact.encode_inbox(ib, None, None)
    assert len(ci.reqs.req) == 0 and int(ci.reqs.op_esc["op_meta"][0]) & 0xFF == abi.COP_MALFORMED
    seen = compact.stands_for(ib)
    model.assert_step_reads_the_same(seen, model.unpack(ci, np.array([3]), model.InFlight(1, 2)))
    o2, _ = _one_group()
    want, got = o.step(ib), o2.step(seen)
    assert abi.ERR_NAMES[(int(want.rep_meta[0, 0]) >> 8) & 0xFF] == "BAD_EVENT"
    harness.assert_outbox_equal(want, got)
    harness.assert_states_equal(o, o2, [0], 2)


def test_an_op_beyond_the_16_bit_offset_travels_as_an_op_escape():
    """Two SUBMITs 70 s apart in one row: op_c's 16-bit offset cannot hold the second, which used to raise ValueError."""
    ib2 = abi.Inbox(1, 2, 2)
    ib2.submit(0, 0, harness.T0)
    ib2.submit(0, 1, harness.T0 + 70_000, unavail=1)
    ci = compact.encode_inbox(ib2, None, None)
    assert ci.op_c[0, 1] == 0 and int(ci.reqs.op_esc["now_ms"][0]) == harness.T0 + 70_000
    model.assert_step_reads_the_same(ib2, model.unpack(ci, np.zeros(2, np.int64), model.InFlight(2, 2)))


def test_a_sweep_rows_dropped_request_leaves_no_unavailable_mask():
    """A request on a sweep row is dropped from the step; its term in op_ab used to be read as an unavailable mask (and one
    of 2^31 or more was refused as a mask beyond 16 lanes)."""
    ib = abi.Inbox(2, 1, 2, ent_cap=1, sweep=True)
    ib.row_now[0] = harness.T0
    ib.vote_request(0, 0, harness.T0, 1, harness.T31, 5, 1)
    ib.submit(1, 0, harness.T0 + 1)
    ci = compact.encode_inbox(ib, None, None, sweep=True)
    assert ci.op_unavail is None and ci.reqs is None


def test_ballot_terms_may_be_given_per_lane():
    """Two lanes of one group answer ballots of different terms in one row: each vote reply travels as a word."""
    ib = abi.Inbox(1, 1, 2)
    ib.vote_reply(0, 0, 0, harness.T0, 0, 7, True)
    ib.vote_reply(0, 0, 1, harness.T0, 0, 9, True)
    bt = np.array([[[7, 9]]], np.int64)
    tags = np.array([[[0, 1]]], np.uint8)
    ci = compact.encode_inbox(ib, None, None, elections=True, ballot_term=bt, ballot_inc=np.zeros((1, 1, 2), np.uint64),
                              ballot_tags=tags)
    assert len(ci.esc) == 0 and ((ci.ev_c >> np.uint32(13)) & np.uint32(7)).tolist() == [[[0, 0]]]


def test_a_wide_append_entries_travels_as_a_record_and_moves_the_commit():
    """An AppendEntries to a group whose log lies near 2^40, with a leader commit two entries above its prevLogIndex: it is a
    compact record (d_commit = 2), the model's unpack rebuilds prev + d_commit in 64 bits, and the step moves the group's
    commit index to it."""
    cfg = abi.make_cfg(replicas=3, max_groups=1, max_rows=1, entry_pool_cap=16)
    o = binding.Oracle(cfg)
    init = harness.wide_init(1, big=[0])
    o.open_bulk(0, init)
    st = o.export(0)
    prev, term = st.last_index, st.current_term
    ib = abi.Inbox(1, 1, 2, ent_cap=4)
    ib.ae_request(0, 0, harness.T0, 1, term, prev, st.last_term, [term, term], leader_commit=prev + 2)
    ci = compact.encode_inbox(ib, None, None)
    assert len(ci.reqs.req) == 1 and len(ci.reqs.op_esc) == 0 and int(ci.reqs.req["d_commit"][0]) == 2
    seen = model.unpack(ci, np.array([term]), model.InFlight(1, 2))
    assert int(seen.op_cd["y"][0, 0]) == prev + 2 > 1 << 40
    model.assert_step_reads_the_same(ib, seen)
    o.step(ib)
    assert o.export(0).commit_index == prev + 2 > st.commit_index
