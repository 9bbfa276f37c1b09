"""Elections through the compact host path, on CPU (RAFTING_COMPACT_ELECTIONS): ballots as plan_c lanes, vote replies as
ev_c words and inbound vote requests as records are lossless.  A numpy restatement of the engine's flagged unpack / pack
kernels (tests/compact_model.py) runs around the oracle on the config #3 vote storm and the config #5 mixed stream:
every dense inbox must survive encode -> unpack on every column the step reads, every dense outbox pack -> decode."""
import numpy as np
import pytest

from oracle import binding
from rafting_b200 import abi, compact, workload
from tests import compact_model as model
from tests import harness
from tests.compact_model import EL, assert_step_reads_the_same

U64 = np.uint64


@pytest.mark.parametrize("rows", [1, 2])
def test_vote_storm_round_trips_through_the_election_words_and_mostly_travels_compact(rows):
    G, R, steps, settle = 256, 5, 16, 2
    F = R - 1
    o, w = model.storm(G, R, rows)
    st = model.InFlight(G, F)
    g_term = np.array([o.export(g).current_term for g in range(G)], dtype=np.int64)
    prev, nxt, ratios = None, None, model.Ratios()
    for k in range(steps):
        ib = workload.vote_inbox_host(w, k, prev)
        ci = model.encode(ib, nxt, EL, empty_list=False)
        assert_step_reads_the_same(ib, model.unpack(ci, g_term, st, EL), where=f"encode -> unpack, step {k}")
        dense = o.step(ib)
        co = model.pack(dense, model.oracle_epoch(o, G), st, esc_cap=rows * G * F + 2 * rows * G, flags=EL, replies=True)
        harness.assert_outbox_equal(dense, compact.decode_outbox(co, elections=True), where=f"pack -> decode, step {k}")
        if k >= settle:
            ratios.add(ib, ci, dense, co)
        prev, nxt, g_term = dense, model.next_of(dense, co), dense.current_term.copy()
    if rows == 1:
        ratios.assert_mostly_compact()
    else:
        # a row's ballot is compact only if it still matches the END of the step: with several rows a later row often moves
        # the group on (a vote storm is carried one row per launch); lossless either way
        assert ratios.ballot_lanes > 0.5 * ratios.ballots and ratios.reply_words > 0.5 * ratios.replies, vars(ratios)
    assert int(st.bits.astype(np.uint64).sum()) > 0                     # ballots hold tags between steps


def test_mixed_stream_round_trips_with_the_flag_and_its_appendentries_stay_as_compact():
    G, R, rows, steps, settle = 256, 3, 4, 40, 8
    F = R - 1
    cfg = abi.make_cfg(replicas=R, max_groups=G, max_rows=rows, entry_pool_cap=workload.POOL_TERMS)
    o = binding.Oracle(cfg)
    o.open_bulk(0, harness.init_array(G, terms=np.arange(G) % 7))
    harness.elect_all(o, workload.make_wl(0x5EED0005, 1, G, F))
    w = workload.make_wl(0x5EED0005, rows, G, F)
    st, st0 = model.InFlight(G, F), model.InFlight(G, F)
    g_term = np.array([o.export(g).current_term for g in range(G)], dtype=np.int64)
    prev, nxt, nxt0 = None, None, None
    flagged, plain = model.Ratios(), model.Ratios()
    for k in range(steps):
        ib = workload.mixed_inbox_host(w, k, prev)
        ci = model.encode(ib, nxt, EL, empty_list=False)
        ci0 = model.encode(ib, nxt0, 0, empty_list=False)                      # the same step without the flag
        assert_step_reads_the_same(ib, model.unpack(ci, g_term, st, EL), where=f"encode -> unpack, step {k}")
        dense = o.step(ib)
        co = model.pack(dense, model.oracle_epoch(o, G), st, esc_cap=rows * G * F + 2 * rows * G, flags=EL, replies=True)
        harness.assert_outbox_equal(dense, compact.decode_outbox(co, elections=True), where=f"pack -> decode, step {k}")
        model.unpack(ci0, g_term, st0)
        co0 = model.pack(dense, model.oracle_epoch(o, G), st0, esc_cap=rows * G * F + 2 * rows * G, replies=True)
        if k >= settle:
            flagged.add(ib, ci, dense, co)
            plain.add(ib, ci0, dense, co0)
        prev, nxt, g_term = dense, model.next_of(dense, co), dense.current_term.copy()
        nxt0 = model.next_of(dense, co0)
    assert flagged.ae > 1000 and flagged.ae_records == plain.ae_records, (vars(flagged), vars(plain))
    assert flagged.ballots > 0 and flagged.ballot_lanes > 0, vars(flagged)         # four rows: many ballots are superseded


def _one_step(o, ib, nxt, st, G, esc_cap=4096):
    ci = model.encode(ib, nxt, EL, empty_list=False)
    assert_step_reads_the_same(ib, model.unpack(ci, np.array([o.export(g).current_term for g in range(G)]), st, EL))
    dense = o.step(ib)
    co = model.pack(dense, model.oracle_epoch(o, G), st, esc_cap=esc_cap, flags=EL, replies=True)
    harness.assert_outbox_equal(dense, compact.decode_outbox(co, elections=True))
    return ci, dense, co


def test_every_rule_a_vote_breaks_sends_it_in_full():
    G, R, rows = 16, 5, 2
    F = R - 1
    cfg = abi.make_cfg(replicas=R, max_groups=G, max_rows=rows, entry_pool_cap=4096)
    o = binding.Oracle(cfg)
    o.open_bulk(0, harness.init_array(G, terms=3, last_index=20, last_term=3, commit_index=10))
    t0 = harness.T0
    st = model.InFlight(G, F)
    # step 1: every group times out in row 0 (PreVote ballot, term 4); group 1 then receives a RequestVote of term 6 in row 1,
    # which replaces its ballot's role object within the step: that ballot no longer matches the end-of-step columns
    ib = abi.Inbox(rows, G, F)
    for g in range(G):
        ib.timeout(0, g, t0)
    ib.vote_request(1, 1, t0 + 5, 0, 6, 20, 3)
    ci, dense, co = _one_step(o, ib, None, st, G)
    assert (dense.ballot_meta[0] != 0).all()
    kinds = co.plan_c[0, :, 0] & np.uint32(7)
    assert kinds[1] == 0 and (np.delete(kinds, 1) == abi.CPLAN_PREVOTE).all()
    esc = co.esc[:int(co.counts[0])]
    assert [(int(r["kind"]), int(r["slot"])) for r in esc if r["kind"] == abi.CESC_BALLOT] == [(abi.CESC_BALLOT, 1)]
    assert ci.reqs is not None and ci.reqs.req["slot"].tolist() == [G + 1] and len(ci.reqs.op_esc) == 0
    nxt = model.next_of(dense, co)
    # step 2: the replies, one rule broken per group
    ib = abi.Inbox(rows, G, F)
    inc = dense.ballot_meta[0] >> U64(32)
    for g in range(G):
        for f in range(F):
            ib.vote_reply(0, g, f, t0 + 20, int(inc[g]), 3, f == 0, pre=True)   # granted by lane 0: no majority
    ib.vote_reply(0, 2, 1, t0 + 20, int(inc[2]), 9, False, pre=True)              # a higher term
    ib.vote_reply(0, 3, 1, t0 + 20, int(inc[3]), 4 - 8, False, pre=True)          # c = 8
    ib.vote_reply(0, 5, 1, t0 + 70_000, int(inc[5]), 3, False, pre=True)          # 70 s after the row's base time
    ib.vote_reply(0, 6, 1, t0 + 20, int(inc[6]), 5, False, outcome=abi.OUT_ERROR, pre=True)   # a term without outcome OK
    ib.vote_reply(0, 7, 1, t0 + 20, int(inc[7]) + 1, 3, False, pre=True)          # not the incarnation that asked
    nxt["ballot_tags"][0, 4, 1] = abi.CTAG_NONE                                          # untagged
    ib.prevote_request(1, 8, t0 + 25, 0, 5, 20, 3)                                # fits: a record
    ib.vote_request(1, 9, t0 + 25, 0, 5, 20, 3, rand=777)                         # an explicit draw
    ib.prevote_request(1, 10, t0 + 25, 0, 2, 20, 3)                               # term < lastLogTerm
    ib.vote_request(1, 11, t0 + 25, 0, 5, 20, 3)
    ib.op_meta[1, 11] |= U64(1 << 16)                                             # an entry count
    ci, dense, co = _one_step(o, ib, nxt, st, G)
    wk = ci.ev_c[0, :, 1] & np.uint32(0xF)
    escaped = [g for g in range(G) if wk[g] == abi.CEV_ESCAPED]
    assert escaped == [1, 2, 3, 4, 5, 6, 7], escaped                              # group 1: its ballot took no tags
    assert ((wk == abi.EV_PV_REPLY) | (wk == abi.CEV_ESCAPED)).all()
    assert sorted({int(s) // F for s in ci.esc["slot"]}) == escaped
    assert ((ci.ev_c[0, :, 1] >> np.uint32(8)) & np.uint32(0xFF))[4] == abi.CTAG_NONE
    assert ci.reqs.req["slot"].tolist() == [G + 8] and ci.reqs.op_esc["slot"].tolist() == [G + 9, G + 10, G + 11]
    # every tag the ballots took came back, through the words and through the escaped words, except the untagged reply's
    held = st.bits != 0
    assert held[4, 1] and int(held.sum()) == 1, np.argwhere(held)


def test_a_ballot_next_to_a_plan_is_escaped_and_a_malformed_vote_record_is_answered_per_op():
    G, R, rows = 8, 3, 1
    F = R - 1
    cfg = abi.make_cfg(replicas=R, max_groups=G, max_rows=rows, entry_pool_cap=64)
    o = binding.Oracle(cfg)
    o.open_bulk(0, harness.init_array(G, terms=3, last_index=20, last_term=3))
    ib = abi.Inbox(rows, G, F)
    for g in range(G):
        ib.timeout(0, g, harness.T0)
    dense = o.step(ib)
    assert (dense.ballot_meta != 0).all()
    dense.plan_meta[0, 3, 1] = abi.PLAN_SKIP_INFLIGHT | (int(dense.incarnation[3]) << 32)   # a plan in the ballot's row
    dense.plan_meta[0, 4, 1] = abi.PLAN_AE | (int(dense.incarnation[4]) << 32)               # one that takes a tag
    dense.plan_epoch[0, 4, 1] = 7; dense.plan_lc[0, 4, 1] = (20, 0); dense.plan_pp[0, 4, 1] = (20, 3)
    st = model.InFlight(G, F)
    co = model.pack(dense, model.oracle_epoch(o, G), st, esc_cap=64, flags=EL, replies=True)
    kinds = co.plan_c[0, :, :] & np.uint32(7)
    assert (kinds[3] != abi.CPLAN_PREVOTE).all() and (kinds[4] != abi.CPLAN_PREVOTE).all()
    assert (np.delete(kinds, [3, 4], axis=0) == abi.CPLAN_PREVOTE).all()
    assert sorted(int(r["slot"]) for r in co.esc[:int(co.counts[0])] if r["kind"] == abi.CESC_BALLOT) == [3, 4]
    assert int(st.bits[3].sum()) == 0 and int(st.bits[4].sum()) == 1 and int(co.counts[1]) == G
    harness.assert_outbox_equal(dense, compact.decode_outbox(co, elections=True), where="ballot next to a plan")
    # a vote reply on the AE plan's lane answers the escaped ballot, not the plan: it travels in full, its escaped word names
    # no tag, and the plan's tag stays taken
    nxt = model.next_of(dense, co)
    assert nxt["tags"][0, 4, 1] < 32 and nxt["ballot_tags"][0, 4, 1] == abi.CTAG_NONE
    ib = abi.Inbox(rows, G, F)
    for f in range(F):
        ib.vote_reply(0, 4, f, harness.T0 + 20, int(dense.ballot_meta[0, 4]) >> 32, 3, False, pre=True)
    ci = model.encode(ib, nxt, EL, empty_list=False)
    assert (ci.ev_c[0, 4] == (abi.CEV_ESCAPED | (abi.CTAG_NONE << 8))).all() and len(ci.esc) == F
    model.unpack(ci, np.full(G, 3, np.int64), st, EL)
    assert int(st.bits[4, 1]) == 1 << int(nxt["tags"][0, 4, 1])
    # vote records the engine must refuse: a count, a d_commit, kind 3; and a vote record in an unflagged step
    ci = compact.CompactInbox(rows, G, F)
    ci.ev_c = None
    req = np.zeros(4, dtype=abi.CREQ)
    req["slot"] = [0, 1, 2, 3]
    req["meta"] = [abi.creq_make(0, 1, 0) | (1 << 11), abi.creq_make(0, 0, 0) | (2 << 11), abi.creq_make(0, 0, 0) | (3 << 11),
                   abi.creq_make(0, 0, 0) | (1 << 11)]
    req["d_commit"] = [0, 5, 0, 0]
    req["term"], req["prev_index"] = 5, 20
    ci.reqs = compact.CompactRequests(req)
    ib = model.unpack(ci, np.full(G, 3, np.int64), model.InFlight(G, F), EL)
    assert [int(ib.op_meta[0, g]) & 0xFF for g in range(4)] == [abi.COP_MALFORMED] * 3 + [abi.OP_PREVOTE_REQ]
    ib0 = model.unpack(ci, np.full(G, 3, np.int64), model.InFlight(G, F))
    assert [int(ib0.op_meta[0, g]) & 0xFF for g in range(4)] == [abi.COP_MALFORMED] * 4


def test_without_the_flag_the_codec_is_unchanged():
    G, R, rows, steps = 64, 5, 2, 6
    o, w = model.storm(G, R, rows)
    prev = None
    for k in range(steps):
        ib = workload.vote_inbox_host(w, k, prev)
        a = compact.encode_inbox(ib, None, None, None)
        b = compact.encode_inbox(ib, None, None, None, elections=False)
        assert a.ev_c.tobytes() == b.ev_c.tobytes() and a.esc.tobytes() == b.esc.tobytes()
        wk = a.ev_c & np.uint32(0xF)
        assert not ((wk == abi.EV_PV_REPLY) | (wk == abi.EV_RV_REPLY)).any()
        assert ((a.ev_c[wk == abi.CEV_ESCAPED]) == abi.CEV_ESCAPED).all()
        if a.reqs is not None:
            assert not (a.reqs.req["meta"] & np.uint32(0xF800)).any()
        prev = o.step(ib)


def test_native_election_writers_match_the_encoder_directly_and_through_the_jni_glue(tmp_path):
    """rafting_acks_to_cinbox_ex / rafting_failures_to_cinbox_ex (vote replies, with a pending entry per ballot lane) and
    rafting_request_to_creq_ex (inbound vote requests) build, word for word and record for record, the compact inbox that
    compact.encode_inbox(elections=True) builds from the same dense config #3 step; then the same through the stand-in JNIEnv."""
    import ctypes as C
    from rafting_b200 import ingest
    from tests import jni_exec
    G, R, rows, steps = 128, 5, 1, 8
    F = R - 1
    o, w = model.storm(G, R, rows)
    st = model.InFlight(G, F)
    pend = ingest.Pending()
    prev, nxt, seq_of, next_seq = None, None, {}, [1] * F
    words = records = escaped = 0

    def recs_of(ib, r):
        """the inbound vote requests of row r as engine-to-engine request records"""
        out = []
        ok = (ib.op_meta[r] & U64(0xFF)).astype(np.int64)
        for g in np.flatnonzero((ok == abi.OP_PREVOTE_REQ) | (ok == abi.OP_VOTE_REQ)):
            q = np.zeros(1, dtype=ingest.REQ_REC)[0]
            q["gid"], q["kind"], q["src_slot"], q["dst_slot"], q["row"] = g, ok[g], (int(ib.op_meta[r, g]) >> 8) & 0xFF, 1, r
            q["term"], q["a"], q["b"] = ib.op_ab[r, g]["x"], ib.op_ab[r, g]["y"], ib.op_cd[r, g]["x"]
            out.append((q, int(ib.op_nr[r, g]["x"])))
        return out

    for k in range(steps):
        ib = workload.vote_inbox_host(w, k, prev)
        want = model.encode(ib, nxt, EL, empty_list=False)
        got = compact.CompactInbox(rows, G, F)
        got.row_base[:] = want.row_base
        got.op_c[:] = want.op_c
        esc = np.zeros(rows * G * F, dtype=abi.CESC_IN)
        n_esc = 0
        ek = (ib.ev_meta & U64(0xF)).astype(np.int64)
        for r in range(rows):
            for f in range(F):
                all_at = [g for g in range(G) if ek[r, g, f] != 0]
                for now in sorted(set(int(ib.ev_tn["y"][r, g, f]) for g in all_at)):   # one drain per (connection, time)
                    at = [g for g in all_at if int(ib.ev_tn["y"][r, g, f]) == now]
                    ok_at = [g for g in at if (int(ib.ev_meta[r, g, f]) >> 4) & 3 == abi.OUT_OK]
                    acks = np.zeros(len(ok_at), dtype=ingest.ACK_REC)
                    for j, g in enumerate(ok_at):
                        acks[j] = (g, ek[r, g, f], (int(ib.ev_meta[r, g, f]) >> 6) & 1, 0, seq_of[(r, g, f)], 0, ib.ev_tn["x"][r, g, f])
                    rc, n_esc, deferred, unknown = pend.acks_to_cinbox(f, acks, now, r, got, esc, n_esc, flags=abi.COMPACT_ELECTIONS)
                    assert rc == 0 and len(deferred) == 0 and unknown == 0
                    failed = [seq_of[(r, g, f)] for g in at if g not in ok_at]
                    rc, n_esc, deferred, unknown = pend.failures_to_cinbox(f, failed, abi.OUT_ERROR, now, r, got, esc, n_esc,
                                                                           flags=abi.COMPACT_ELECTIONS)
                    assert rc == 0 and len(deferred) == 0 and unknown == 0
        assert len(pend) == 0                                                    # every ballot lane was answered
        assert np.array_equal(got.ev_c, want.ev_c), f"step {k}: ev_c words differ"
        a, b = np.sort(esc[:n_esc], order="slot"), np.sort(want.esc, order="slot")
        assert a.tobytes() == b.tobytes(), f"step {k}: escape records differ"
        place = ingest.CReqPlacer(rows * G, rows * G, 1)
        for r in range(rows):
            for q, now in recs_of(ib, r):
                assert place.put(q, [], r, now, False, got, G, flags=abi.COMPACT_ELECTIONS) == 0
        if want.reqs is not None:
            p = place.requests()
            assert p.req.tobytes() == want.reqs.req.tobytes() and p.op_esc.tobytes() == want.reqs.op_esc.tobytes()
            records += len(p.req)
        words += int(((want.ev_c & np.uint32(0xF)) == abi.EV_PV_REPLY).sum() + ((want.ev_c & np.uint32(0xF)) == abi.EV_RV_REPLY).sum())
        escaped += n_esc
        model.unpack(want, np.zeros(G, np.int64), st, EL)                    # frees the tags the replies answer
        dense = o.step(ib)
        co = model.pack(dense, model.oracle_epoch(o, G), st, esc_cap=rows * G * F + 2 * rows * G, flags=EL, replies=True)
        prev, nxt = dense, model.next_of(dense, co)
        seq_of = {}
        for r, g in np.argwhere(dense.ballot_meta != 0):                        # the ballot leaves on every lane
            r, g = int(r), int(g)
            bm = int(dense.ballot_meta[r, g])
            for f in range(F):
                seq_of[(r, g, f)] = next_seq[f]
                pend.put(f, next_seq[f], abi.EV_PV_REPLY if (bm & 0xF) == abi.BALLOT_PREVOTE else abi.EV_RV_REPLY, g, f,
                         int(nxt["ballot_tags"][r, g, f]), bm >> 32, int(dense.ballot_term[r, g]), 0, 0)
                next_seq[f] += 1
    assert words > 1000 and records > 100 and escaped > 10, (words, records, escaped)
    # the three natives through the JNI glue, on the last step
    L = jni_exec.build(str(tmp_path))
    if L is None:
        pytest.skip("no gcc")
    from tests.jni_exec import Buf, buf_of_array, buf_of_struct, fn
    L.fake_reset()
    place2 = ingest.CReqPlacer(rows * G, rows * G, 1)
    put = fn(L, "requestToCreqEx", None, C.POINTER(Buf), C.POINTER(Buf), C.c_int32, C.c_int64, C.c_uint8, C.POINTER(Buf), C.c_int32,
             C.POINTER(Buf), C.c_int32, C.c_int32, C.c_int32, C.c_int32)
    empty = np.zeros(1, np.int64)
    for q, now in recs_of(ib, 0):
        put(C.byref(buf_of_array(np.array([q], dtype=ingest.REQ_REC))), C.byref(buf_of_array(empty)), 0, now, 0,
            C.byref(buf_of_struct(got.as_c())), G, C.byref(buf_of_struct(place2.c)), *place2.caps, abi.COMPACT_ELECTIONS)
    assert L.fake_throws() == 0, L.fake_thrown_message()
    assert place2.requests().req.tobytes() == want.reqs.req.tobytes()
    # one vote reply and one time-out, each on a fresh pending entry, into an empty row
    got2 = compact.CompactInbox(rows, G, F)
    got2.row_base[:] = want.row_base
    n0 = len(pend)                                                              # the last step's ballots are still out
    pend.put(0, 9001, abi.EV_PV_REPLY, 5, 0, 7, 3, 40, 0, 0)
    pend.put(1, 9002, abi.EV_RV_REPLY, 5, 1, 9, 3, 40, 0, 0)
    acks = np.zeros(1, dtype=ingest.ACK_REC)
    acks[0] = (5, abi.EV_PV_REPLY, 1, 0, 9001, 0, 38)
    counters = np.zeros(3, np.int64)
    esc2, dfr = np.zeros(4, dtype=abi.CESC_IN), np.zeros(4, np.uint32)
    fn(L, "acksToCinboxEx", None, C.c_int64, C.c_int32, C.POINTER(Buf), C.c_int32, C.c_int64, C.c_int32, C.POINTER(Buf), C.c_int32, C.c_int32,
       C.POINTER(Buf), C.c_int32, C.POINTER(Buf), C.POINTER(Buf), C.c_int32)(
        pend._h.value, 0, C.byref(buf_of_array(acks)), 1, int(want.row_base[0]) + 3, 0, C.byref(buf_of_struct(got2.as_c())), G, F,
        C.byref(buf_of_array(esc2)), len(esc2), C.byref(buf_of_array(dfr)), C.byref(buf_of_array(counters)), abi.COMPACT_ELECTIONS)
    fn(L, "failuresToCinboxEx", None, C.c_int64, C.c_int32, C.POINTER(Buf), C.c_int32, C.c_int32, C.c_int64, C.c_int32, C.POINTER(Buf), C.c_int32,
       C.c_int32, C.POINTER(Buf), C.c_int32, C.POINTER(Buf), C.POINTER(Buf), C.c_int32)(
        pend._h.value, 1, C.byref(buf_of_array(np.array([9002], np.int32))), 1, abi.OUT_CANCELED, int(want.row_base[0]) + 4, 0,
        C.byref(buf_of_struct(got2.as_c())), G, F, C.byref(buf_of_array(esc2)), len(esc2), C.byref(buf_of_array(dfr)),
        C.byref(buf_of_array(counters)), abi.COMPACT_ELECTIONS)
    assert L.fake_throws() == 0, L.fake_thrown_message()
    assert int(got2.ev_c[0, 5, 0]) == abi.cev_vote_make(abi.EV_PV_REPLY, abi.OUT_OK, 1, 7, 2, 3)
    assert int(got2.ev_c[0, 5, 1]) == abi.cev_vote_make(abi.EV_RV_REPLY, abi.OUT_CANCELED, 0, 9, 0, 4)
    assert counters.tolist() == [0, 0, 0] and len(pend) == n0
