"""AE plans with an older prevLogTerm through the compact host path, on CPU (RAFTING_COMPACT_PREV_TERM): a numpy restatement of
the flagged pack_kernel (tests/compact_model.py) runs around the oracle on the config #3 vote storm and the config #5
mixed stream with flags 4 and 5.  Every dense outbox must survive pack -> decode, every dense inbox (acks to kind-7 plans
included) encode -> unpack.  rafting_coutbox_to_requests must emit what rafting_outbox_to_requests emits for the decoded
outbox, for every flags value a step may carry."""
import ctypes as C

import numpy as np
import pytest

from oracle import binding
from rafting_b200 import abi, compact, ingest, workload
from tests import compact_model as model
from tests import harness
from tests.compact_model import EL, PT

U64 = np.uint64


class Pump:
    """The host side of one compact stream begun with `flags`, around the model: its in-flight table, and what the next
    step's encoder keeps from the last one."""

    def __init__(self, G, F, flags):
        self.G, self.F, self.flags = G, F, flags
        self.st = model.InFlight(G, F)
        self.nxt = None

    def step(self, o, ib, g_term, where):
        ci = model.encode(ib, self.nxt, self.flags, empty_list=True)
        model.assert_step_reads_the_same(ib, model.unpack(ci, g_term, self.st, self.flags), where=f"encode -> unpack, {where}")
        dense = o.step(ib)
        co = model.pack(dense, model.oracle_epoch(o, self.G), self.st, esc_cap=1 << 20, flags=self.flags, replies=True)
        harness.assert_outbox_equal(dense, compact.decode_outbox(co, elections=bool(self.flags & EL), prev_term=bool(self.flags & PT)),
                                    where=f"pack -> decode, {where}")
        self.nxt = model.next_of(dense, co)
        return ci, dense, co


class Counts:
    """AE plans, how they travelled, and acks that answered a kind-7 word."""

    def __init__(self, G, F):
        self.ae = self.ae_words = self.kind7 = self.plan_records = self.acks_to_kind7 = 0
        self.held7 = np.zeros((G, F, 32), bool)                                   # tags taken by kind-7 words, not yet answered

    def add(self, ci, dense, co, count=True):
        if ci.ev_c is not None:                                                   # acks in this step's inbox
            w = ci.ev_c
            ack = ((w & np.uint32(0xF)) == abi.EV_AE_ACK)
            for r, g, f in np.argwhere(ack):
                tag = (int(w[r, g, f]) >> 8) & 0xFF
                if tag < 32 and self.held7[g, f, tag]:
                    self.held7[g, f, tag] = False
                    self.acks_to_kind7 += count
        k = co.plan_c & np.uint32(7)
        for r, g, f in np.argwhere(k == abi.CPLAN_AE_PREV_TERM):
            tag = (int(co.plan_c[r, g, f]) >> 5) & 63
            if tag < 32:
                self.held7[g, f, tag] = True
        if not count:
            return
        self.ae += int(((dense.plan_meta & U64(0xF)) == abi.PLAN_AE).sum())
        esc = ((co.plan_c >> np.uint32(4)) & np.uint32(1)) != 0
        self.ae_words += int((((k == abi.PLAN_AE) & ~esc) | (k == abi.CPLAN_AE_PREV_TERM)).sum())
        self.kind7 += int((k == abi.CPLAN_AE_PREV_TERM).sum())
        self.plan_records += sum(int(r["kind"]) == abi.CESC_PLAN for r in co.esc[:int(co.counts[0])])


def _unflagged_twin(co, flags):
    """plan_c of the same step without PREV_TERM: every kind-7 word was an escaped kind-1 word with the same tag"""
    k = co.plan_c & np.uint32(7)
    is7 = k == abi.CPLAN_AE_PREV_TERM
    keep = np.uint32(0x8 | (63 << 5))                                            # heartbeat and tag
    return np.where(is7, (co.plan_c & keep) | np.uint32(abi.PLAN_AE | 0x10), co.plan_c)


@pytest.mark.parametrize("flags", [PT, EL | PT])
@pytest.mark.parametrize("rows", [1, 2])
def test_vote_storm_round_trips_and_new_leaders_heartbeats_travel_as_words(rows, flags):
    G, R, steps, settle = 512, 5, 16, 2
    F = R - 1
    o, w = model.storm(G, R, rows)
    flagged, plain = Pump(G, F, flags), Pump(G, F, flags & EL)
    o0, _ = model.storm(G, R, rows)
    g_term = np.array([o.export(g).current_term for g in range(G)], dtype=np.int64)
    cnt, cnt0 = Counts(G, F), Counts(G, F)
    prev = None
    for k in range(steps):
        ib = workload.vote_inbox_host(w, k, prev)
        ci, dense, co = flagged.step(o, ib, g_term, f"step {k}")
        ci0, dense0, co0 = plain.step(o0, ib, g_term, f"unflagged step {k}")
        # the flag changes nothing but the words of the plans it carries: same tags, same inbox encoding
        assert not ((co0.plan_c & np.uint32(7)) == abi.CPLAN_AE_PREV_TERM).any()
        assert np.array_equal(_unflagged_twin(co, flags), co0.plan_c), f"step {k}"
        assert np.array_equal(ci.ev_c, ci0.ev_c) and np.array_equal(flagged.st.bits, plain.st.bits), f"step {k}"
        cnt.add(ci, dense, co, k >= settle)
        cnt0.add(ci0, dense0, co0, k >= settle)
        prev, g_term = dense, dense.current_term.copy()
    assert cnt.kind7 > 100 and cnt.plan_records < cnt0.plan_records, (vars(cnt), vars(cnt0))   # the storm carries no acks
    if rows == 1 and flags == EL | PT:
        assert cnt.ae_words >= 0.95 * cnt.ae, vars(cnt)


@pytest.mark.parametrize("flags", [PT, EL | PT])
def test_mixed_stream_round_trips_and_halves_its_plan_records(flags):
    G, R, rows, steps, settle = 256, 3, 4, 40, 8
    F = R - 1
    pumps, oracles = [], []
    for fl in (flags, flags & EL):
        cfg = abi.make_cfg(replicas=R, max_groups=G, max_rows=rows, entry_pool_cap=workload.POOL_TERMS)
        o = binding.Oracle(cfg)
        o.open_bulk(0, harness.init_array(G, terms=np.arange(G) % 7))
        harness.elect_all(o, workload.make_wl(0x5EED0005, 1, G, F))
        pumps.append(Pump(G, F, fl)); oracles.append(o)
    w = workload.make_wl(0x5EED0005, rows, G, F)
    g_term = np.array([oracles[0].export(g).current_term for g in range(G)], dtype=np.int64)
    cnt, cnt0 = Counts(G, F), Counts(G, F)
    prev = None
    for k in range(steps):
        ib = workload.mixed_inbox_host(w, k, prev)
        ci, dense, co = pumps[0].step(oracles[0], ib, g_term, f"step {k}")
        ci0, dense0, co0 = pumps[1].step(oracles[1], ib, g_term, f"unflagged step {k}")
        assert np.array_equal(_unflagged_twin(co, flags), co0.plan_c), f"step {k}"
        cnt.add(ci, dense, co, k >= settle)
        cnt0.add(ci0, dense0, co0, k >= settle)
        prev, g_term = dense, dense.current_term.copy()
    assert cnt0.plan_records > 500 and cnt.plan_records <= 0.5 * cnt0.plan_records, (vars(cnt), vars(cnt0))
    assert cnt.acks_to_kind7 > 100, vars(cnt)


def _rules_case():
    """One oracle step of 16 leaders with a plan on lane 1 of every group, then plan fields set by hand: one rule per group."""
    G, R, rows = 16, 3, 1
    F = R - 1
    cfg = abi.make_cfg(replicas=R, max_groups=G, max_rows=rows, entry_pool_cap=4096)
    o = binding.Oracle(cfg)
    o.open_bulk(0, harness.init_array(G, terms=3, last_index=400, last_term=3, commit_index=300))
    harness.elect_all(o, workload.make_wl(0x5EED0005, 1, G, F))
    dense = o.step(abi.Inbox(rows, G, F))
    ep = model.oracle_epoch(o, G)
    for name in ("plan_meta", "plan_pp", "plan_lc", "plan_epoch"):
        getattr(dense, name)[...] = 0
    term, last, commit, inc = dense.current_term, dense.last_entry["x"], dense.commit_index, dense.incarnation

    def plan(g, gap=2, dprev=3, count=2, dcommit=5, inc_d=0, ep_d=0, last_d=0, hb=0):
        prev = int(last[g]) - dprev
        dense.plan_meta[0, g, 1] = abi.PLAN_AE | (hb << 4) | (count << 16) | ((int(inc[g]) + inc_d) << 32)
        dense.plan_pp[0, g, 1] = (prev, int(term[g]) - gap)
        dense.plan_lc[0, g, 1] = (prev + count + last_d, int(commit[g]) - dcommit)
        dense.plan_epoch[0, g, 1] = int(ep[g]["x"]) + ep_d

    cases = {0: dict(), 1: dict(gap=8), 2: dict(gap=9), 3: dict(gap=0), 4: dict(dcommit=15), 5: dict(dcommit=16),
             6: dict(dprev=255), 7: dict(dprev=256), 8: dict(inc_d=1), 9: dict(ep_d=1), 10: dict(last_d=1),
             11: dict(count=0, dprev=0, dcommit=0, hb=1), 12: dict(gap=0, dcommit=100), 13: dict(count=63, gap=1)}
    for g, kw in cases.items():
        plan(g, **kw)
    return dense, ep, G, F


def test_every_rule_a_plan_breaks_sends_it_in_full():
    dense, ep, G, F = _rules_case()
    for flags in (PT, EL | PT):
        st = model.InFlight(G, F)
        co = model.pack(dense, ep, st, esc_cap=64, flags=flags, replies=True)
        k = (co.plan_c[0, :, 1] & np.uint32(7)).tolist()
        escaped = ((co.plan_c[0, :, 1] >> np.uint32(4)) & np.uint32(1)).tolist()
        seven, one = abi.CPLAN_AE_PREV_TERM, abi.PLAN_AE
        assert [k[g] for g in (0, 1, 4, 6, 11, 13)] == [seven] * 6, k                  # every rule at its limit: a word
        assert [k[g] for g in (3, 12)] == [one, one] and escaped[3] == escaped[12] == 0    # gap 0: kind 1, its dcommit < 128
        assert [(k[g], escaped[g]) for g in (2, 5, 7, 8, 9, 10)] == [(one, 1)] * 6, (k, escaped)   # one rule broken: a record
        recs = sorted(int(r["slot"]) // F for r in co.esc[:int(co.counts[0])] if r["kind"] == abi.CESC_PLAN)
        assert recs == [2, 5, 7, 8, 9, 10], recs
        w = int(co.plan_c[0, 1, 1])
        assert ((w >> 25) & 7) + 1 == 8 and (w >> 28) == 5 and (w >> 17) & 255 == 3 and (w >> 11) & 63 == 2
        assert (int(co.plan_c[0, 11, 1]) >> 3) & 1 == 1                              # heartbeat bit
        # every plan took a tag, kind 7 and escaped ones alike
        assert (co.tags(rpc_only=True)[0, :14, 1] < 32).all() and (st.bits[:14, 1] == 1).all()
        harness.assert_outbox_equal(dense, compact.decode_outbox(co, elections=bool(flags & EL), prev_term=True), where=f"flags {flags}")
        # without the flag the same outbox never holds kind 7, and its words are those of the model without the flag
        st0 = model.InFlight(G, F)
        co0 = model.pack(dense, ep, st0, esc_cap=64, flags=flags & EL, replies=True)
        assert not ((co0.plan_c & np.uint32(7)) == seven).any()
        assert np.array_equal(_unflagged_twin(co, flags), co0.plan_c)


def _dispatch_pair(G, F, local_slot):
    return ingest.Dispatch(G, F, local_slot), ingest.Dispatch(G, F, local_slot)


def _expected_tags(recs, co, flags, local_slot):
    """the tag a pump puts into each record's pending entry, from the compact outbox's own columns"""
    at = co.tags(rpc_only=True)
    bt = co.ballot_tags() if flags & EL else np.full(co.plan_c.shape, abi.CTAG_NONE, np.uint8)
    out = []
    for q in recs:
        f = int(q["dst_slot"]) if int(q["dst_slot"]) < local_slot else int(q["dst_slot"]) - 1
        vote = int(q["kind"]) in (abi.OP_PREVOTE_REQ, abi.OP_VOTE_REQ)
        out.append(int((bt if vote else at)[int(q["row"]), int(q["gid"]), f]))
    return out


def _check_dispatch(d_dense, d_comp, co, rows, flags, local_slot, rng, where):
    want, unk = d_dense.requests(compact.decode_outbox(co, elections=bool(flags & EL), prev_term=bool(flags & PT)), rows)
    n = int(co.counts[0])
    co.esc[:n] = co.esc[:n][rng.permutation(n)]                                 # the engine's list order is arbitrary
    got, tags, unk2 = d_comp.crequests(co, rows, flags)
    assert got.tobytes() == want.tobytes() and unk == unk2, where
    assert tags.tolist() == _expected_tags(got, co, flags, local_slot), where
    return len(got)


@pytest.mark.parametrize("flags", [0, EL, PT, EL | PT])
def test_coutbox_to_requests_matches_the_dense_dispatch_on_both_streams(flags):
    rng = np.random.default_rng(7)
    # config #3 storm, one row
    G, R, rows = 256, 5, 1
    F = R - 1
    o, w = model.storm(G, R, rows)
    p = Pump(G, F, flags)
    dd, dc = _dispatch_pair(G, F, 1)
    g_term = np.array([o.export(g).current_term for g in range(G)], dtype=np.int64)
    prev, total = None, 0
    for k in range(10):
        ib = workload.vote_inbox_host(w, k, prev)
        _, dense, co = p.step(o, ib, g_term, f"storm step {k}")
        total += _check_dispatch(dd, dc, co, rows, flags, 1, rng, f"storm step {k}")
        prev, g_term = dense, dense.current_term.copy()
    assert total > 1000
    # config #5, four rows
    G, R, rows = 128, 3, 4
    F = R - 1
    cfg = abi.make_cfg(replicas=R, max_groups=G, max_rows=rows, entry_pool_cap=workload.POOL_TERMS)
    o = binding.Oracle(cfg)
    o.open_bulk(0, harness.init_array(G, terms=np.arange(G) % 7))
    harness.elect_all(o, workload.make_wl(0x5EED0005, 1, G, F))
    w = workload.make_wl(0x5EED0005, rows, G, F)
    p = Pump(G, F, flags)
    dd, dc = _dispatch_pair(G, F, 0)
    g_term = np.array([o.export(g).current_term for g in range(G)], dtype=np.int64)
    prev, total = None, 0
    for k in range(24):
        ib = workload.mixed_inbox_host(w, k, prev)
        _, dense, co = p.step(o, ib, g_term, f"config #5 step {k}")
        total += _check_dispatch(dd, dc, co, rows, flags, 0, rng, f"config #5 step {k}")
        prev, g_term = dense, dense.current_term.copy()
    assert total > 1000


def test_coutbox_to_requests_refuses_overflow_and_unknown_flags_and_the_writers_take_bit_4(tmp_path):
    dense, ep, G, F = _rules_case()
    co = model.pack(dense, ep, model.InFlight(G, F), esc_cap=64, flags=PT, replies=True)
    d = ingest.Dispatch(G, F, 0)
    recs, tags, unknown = d.crequests(co, 1, PT)
    assert len(recs) == 13 and unknown == 1 and tags.tolist() == [0] * 13     # group 8's plan names an unseen incarnation
    assert [int(q["b"]) for q in recs[:3]] == [int(dense.current_term[g]) - gap for g, gap in ((0, 2), (1, 8), (2, 9))]
    for bad in (2, 8, 16, 0x80000000):
        with pytest.raises(ValueError):
            d.crequests(co, 1, bad)
    with pytest.raises(ValueError):
        d.crequests(co, 1, PT, cap=3)                                           # no room: RAFTING_E_CAPACITY
    full = compact.CompactOutbox(1, G, F, esc_cap=2)
    for name in compact.CompactOutbox.COLS:
        getattr(full, name)[...] = getattr(co, name)
    full.counts[:] = co.counts
    assert int(full.counts[0]) > 2
    with pytest.raises(OverflowError):
        d.crequests(full, 1, PT)
    # the three writers accept bit 4 (and still refuse bit 2)
    cin = compact.CompactInbox(1, G, F)
    pend = ingest.Pending()
    esc = np.zeros(8, dtype=abi.CESC_IN)
    for flags, rc_want in ((PT, 0), (EL | PT, 0), (2, -1), (8, -1)):
        pend.put(0, 5, abi.EV_AE_ACK, 3, 0, 4, int(dense.incarnation[3]), int(dense.current_term[3]), 0, 0)
        acks = np.zeros(1, dtype=ingest.ACK_REC)
        acks[0] = (3, abi.EV_AE_ACK, 1, 0, 5, 0, int(dense.current_term[3]))
        cin.ev_c[...] = 0
        rc, _, _, _ = pend.acks_to_cinbox(0, acks, 0, 0, cin, esc, 0, flags=flags)
        assert rc == rc_want, flags
        if rc == 0:
            assert int(cin.ev_c[0, 3, 0]) == abi.CEV_ESCAPED or (int(cin.ev_c[0, 3, 0]) >> 8) & 0xFF == 4
        pend.put(0, 6, abi.EV_AE_ACK, 3, 1, 4, 0, 0, 0, 0)
        cin.ev_c[...] = 0
        rc, _, _, _ = pend.failures_to_cinbox(0, [6], abi.OUT_ERROR, 0, 0, cin, esc, 0, flags=flags)
        assert rc == rc_want, flags
        pend.remove(0, 5), pend.remove(0, 6)
        place = ingest.CReqPlacer(4, 4, 4)
        q = np.zeros(1, dtype=ingest.REQ_REC)[0]
        q["gid"], q["kind"], q["src_slot"], q["term"], q["a"], q["b"] = 2, abi.OP_AE_REQUEST, 1, 5, 10, 5
        assert place.put(q, [], 0, 0, False, cin, G, flags=flags) == rc_want, flags


def test_coutbox_to_requests_through_the_jni_glue(tmp_path):
    from tests import jni_exec
    L = jni_exec.build(str(tmp_path))
    if L is None:
        pytest.skip("no gcc")
    from tests.jni_exec import Buf, buf_of_array, buf_of_struct, fn
    dense, ep, G, F = _rules_case()
    co = model.pack(dense, ep, model.InFlight(G, F), esc_cap=64, flags=EL | PT, replies=True)
    want, want_tags, _ = ingest.Dispatch(G, F, 0).crequests(co, 1, EL | PT)
    d = ingest.Dispatch(G, F, 0)
    recs, tags = np.zeros(64, dtype=ingest.REQ_REC), np.zeros(64, np.uint8)
    call = fn(L, "coutboxToRequests", C.c_int32, C.c_int64, C.POINTER(Buf), C.c_int32, C.c_int32, C.POINTER(Buf), C.POINTER(Buf), C.c_int32)
    L.fake_reset()
    n = call(d._h.value, C.byref(buf_of_struct(co.as_c())), 1, EL | PT, C.byref(buf_of_array(recs)), C.byref(buf_of_array(tags)), 64)
    assert L.fake_throws() == 0, L.fake_thrown_message()
    assert n == len(want) and recs[:n].tobytes() == want.tobytes() and np.array_equal(tags[:n], want_tags)
    call(d._h.value, C.byref(buf_of_struct(co.as_c())), 1, 8, C.byref(buf_of_array(recs)), C.byref(buf_of_array(tags)), 64)
    assert L.fake_throws() == 1 and b"IllegalArgument" in L.fake_thrown_class()
