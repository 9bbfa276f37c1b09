"""Inbound requests through the compact host path, on CPU: the request list (rafting_creqs_t) and the compact replies in
rep_c are lossless.  The numpy restatement of the engine's unpack / pack kernels (tests/compact_model.py) runs around the
oracle on the config #5 mixed stream (leader churn, AppendEntries to followers, InstallSnapshot catch-up, flushes, elections):
every dense inbox must survive encode -> unpack on every column the step reads, every dense outbox pack -> decode."""
import ctypes as C

import numpy as np
import pytest

from oracle import binding
from rafting_b200 import abi, compact, workload
from tests import compact_model as model
from tests import harness

U64 = np.uint64
E_INVAL = -1


def test_mixed_stream_round_trips_through_the_request_list_and_mostly_travels_compact():
    G, R, rows, steps, settle = 256, 3, 4, 48, 8                        # 192 ticks: a full 64-tick churn and 128-tick catch-up cycle
    F = R - 1
    cfg = abi.make_cfg(replicas=R, max_groups=G, max_rows=rows, entry_pool_cap=workload.POOL_TERMS)
    o = binding.Oracle(cfg)
    o.open_bulk(0, harness.init_array(G, terms=np.arange(G) % 7))
    harness.elect_all(o, workload.make_wl(0x5EED0005, 1, G, F))
    w = workload.make_wl(0x5EED0005, rows, G, F)
    st = model.InFlight(G, F)
    g_term = np.array([o.export(g).current_term for g in range(G)], dtype=np.int64)
    prev, nxt = None, None
    ae = records = valid = compact_replies = 0
    kinds = set()
    for k in range(steps):
        ib = workload.mixed_inbox_host(w, k, prev)
        ci = model.encode(ib, nxt, 0, empty_list=False)
        model.assert_step_reads_the_same(ib, model.unpack(ci, g_term, st), where=f"encode -> unpack, step {k}")
        dense = o.step(ib)
        co = model.pack(dense, model.oracle_epoch(o, G), st, esc_cap=rows * G * F + 2 * rows * G, replies=True)
        harness.assert_outbox_equal(dense, compact.decode_outbox(co), where=f"pack -> decode, step {k}")
        kinds |= set((ib.op_meta & U64(0xFF)).ravel().tolist())
        if k >= settle:
            ae += int(((ib.op_meta & U64(0xFF)) == abi.OP_AE_REQUEST).sum())
            records += 0 if ci.reqs is None else len(ci.reqs.req)
            valid += int((dense.rep_meta & 1).sum())
            compact_replies += int((co.rep_c >> 7).sum())
        prev, nxt = dense, model.next_of(dense, co)
        g_term = dense.current_term.copy()
    assert {abi.OP_AE_REQUEST, abi.OP_FLUSH, abi.OP_SUBMIT, abi.OP_TIMEOUT} <= kinds
    assert ae > 1000 and valid > 1000, (ae, valid)
    assert records >= 0.9 * ae, (records, ae)
    assert compact_replies >= 0.9 * valid, (compact_replies, valid)


def test_every_rule_a_request_breaks_sends_it_in_full():
    G, R, rows = 16, 3, 2
    F = R - 1
    cfg = abi.make_cfg(replicas=R, max_groups=G, max_rows=rows, entry_pool_cap=4096)
    o = binding.Oracle(cfg)
    o.open_bulk(0, harness.init_array(G, terms=3, last_index=20, last_term=3, commit_index=10))
    t0 = harness.T0
    ib = abi.Inbox(rows, G, F, ent_cap=256)
    ib.ae_request(0, 0, t0, 1, 3, 20, 3, [3, 3], leader_commit=12)                   # fits: a record
    ib.ae_request(0, 1, t0, 1, 3, 20, 3, [3, 2], leader_commit=12)                   # an entry term differs from the request's
    ib.ae_request(0, 2, t0, 1, 3, 20, 3, [3], leader_commit=12, first_index=23)      # op_e != prev + 1
    ib.ae_request(0, 3, t0, 1, 3, 20, 3, [3], leader_commit=12, rand=1234)           # an explicit draw
    ib.ae_request(0, 4, t0, 1, 3, 20, 4, [3], leader_commit=12)                      # term < prevLogTerm
    ib.ae_request(0, 5, t0, 1, 3, 20, 3, [3], leader_commit=20 + (1 << 31))          # leaderCommit - prev beyond int32
    ib.ae_request(0, 6, t0 + 70_000, 1, 3, 20, 3, [3], leader_commit=12)             # 70 s after the row's base time
    ib.prevote_request(0, 7, t0, 2, 4, 20, 3)
    ib.vote_request(0, 8, t0, 2, 4, 20, 3)
    ib.is_request(0, 9, t0, 1, 3, 30, 3, True)
    ib.flush(0, 10, t0, 5, 3)
    ib.timeout(0, 11, t0, rand=1500)                                                 # SUBMIT / TIMEOUT with a draw
    ib.submit(0, 12, t0, count=2)                                                    # stays an op_c word
    ib.ae_request(1, 0, t0 + 5, 1, 3, 22, 3, [], leader_commit=22)                   # heartbeat: a record without entries
    ib.ae_request(1, 1, t0 + 5, 1, 3, 20, 3, [3] * 64, leader_commit=12)             # 64 entries: more than a record holds
    ci = compact.encode_inbox(ib, None, None, None)
    assert sorted(ci.reqs.req["slot"].tolist()) == [0, G]
    assert ci.reqs.op_esc["slot"].tolist() == list(range(1, 12)) + [G + 1]
    assert ci.reqs.req_entries == 2 and len(ci.reqs.ent_terms) == 2 + 5 + 64            # the escapes' terms
    assert int(ci.op_c[0, 12]) & 0xF == abi.OP_SUBMIT and not (ci.op_c[0, :12] & 0xF).any()
    st = model.InFlight(G, F)
    model.assert_step_reads_the_same(ib, model.unpack(ci, np.full(G, 3, np.int64), st), where="forced escapes")
    dense = o.step(ib)
    co = model.pack(dense, model.oracle_epoch(o, G), st, esc_cap=256, replies=True)
    harness.assert_outbox_equal(dense, compact.decode_outbox(co), where="forced escapes")
    assert (dense.rep_meta & 1).sum() >= 10


def test_a_step_without_requests_encodes_as_before():
    G, R, rows = 64, 3, 4
    w = workload.make_wl(11, rows, G, R - 1)
    ib = workload.leader_inbox_host(w, 0, None)
    ci = compact.encode_inbox(ib, None, None, None)
    assert ci.reqs is None
    st = model.InFlight(G, R - 1)
    back = model.unpack(ci, np.zeros(G, np.int64), st)
    assert back.flags == abi.INBOX_NO_REQUESTS and back.op_cd is None


def test_native_placement_and_replies_match_the_encoder_and_the_dense_helpers(tmp_path):
    """rafting_request_to_creq / rafting_coutbox_to_replies against the numpy encoder / decoder and the dense
    rafting_request_to_inbox / rafting_outbox_to_replies, on request records a leader's outboxes produce
    (rafting_outbox_to_requests), placed at a follower node; then the same through the JNI glue's stand-in JNIEnv."""
    from rafting_b200 import ingest
    from tests import jni_exec
    G, R, rows = 128, 3, 4
    F = R - 1
    cfg_a = abi.make_cfg(replicas=R, max_groups=G, max_rows=rows, local_slot=0)
    cfg_b = abi.make_cfg(replicas=R, max_groups=G, max_rows=rows, local_slot=1, entry_pool_cap=rows * G * 64)
    a, b = binding.Oracle(cfg_a), binding.Oracle(cfg_b)
    init = harness.init_array(G, terms=np.arange(G) % 7)
    a.open_bulk(0, init), b.open_bulk(0, init)
    harness.elect_all(a, workload.make_wl(21, 1, G, F))
    w = workload.make_wl(21, rows, G, F)
    disp = ingest.Dispatch(G, F, 0)
    st = model.InFlight(G, F)
    prev, checked, escaped, compact_replies = None, 0, 0, 0
    for k in range(6):
        prev = a.step(workload.leader_inbox_host(w, k, prev))
        recs, unknown = disp.requests(prev, rows)
        recs = recs[recs["dst_slot"] == 1]
        assert unknown == 0 and len(recs) > 0
        terms_of = []
        for j, q in enumerate(recs):
            t = np.full(int(q["count"]) if q["kind"] == abi.OP_AE_REQUEST else 0, int(q["term"]), np.int64)
            if j % 7 == 3 and len(t):
                t[0] -= 1                                                       # an entry of an older term: the request escapes
            terms_of.append(t)
        now = lambda r: harness.T0 + 1000 * k + r
        dense = abi.Inbox(rows, G, F, ent_cap=rows * G * 64, with_events=False)
        for q, t in zip(recs, terms_of):
            assert ingest.request_to_inbox(q, t, int(q["row"]), now(int(q["row"])), False, dense) == 0
        cin = compact.encode_inbox(dense, None, None, None)
        place = ingest.CReqPlacer(rows * G, rows * G, rows * G * 64)
        for q, t in zip(recs, terms_of):
            assert place.put(q, t, int(q["row"]), now(int(q["row"])), False, cin, G) == 0
        assert place.put(recs[0], terms_of[0], int(recs[0]["row"]), now(0), False, cin, G) == E_INVAL      # the slot is taken
        got, want = place.requests(), cin.reqs
        assert got.req.tobytes() == want.req.tobytes() and got.op_esc.tobytes() == want.op_esc.tobytes()
        assert np.array_equal(got.ent_terms, want.ent_terms) and got.req_entries == want.req_entries
        escaped += len(got.op_esc)
        out = b.step(dense)
        co = model.pack(out, model.oracle_epoch(b, G), st, esc_cap=rows * G * 2, replies=True)
        prow = recs["row"].astype(np.uint8)
        rd = ingest.outbox_to_replies(out, G, 1, recs, prow)
        rc = ingest.coutbox_to_replies(co, G, 1, recs, prow)
        assert len(rd) > 0 and rd.tobytes() == rc.tobytes()
        checked += len(rd)
        compact_replies += int((co.rep_c >> 7).sum())
    assert checked > 500 and escaped > 50 and compact_replies > 0.9 * checked
    # the two natives through the JNI glue
    L = jni_exec.build(str(tmp_path))
    if L is None:
        pytest.skip("no gcc")
    from tests.jni_exec import Buf, buf_of_array, buf_of_struct, fn
    place2 = ingest.CReqPlacer(rows * G, rows * G, rows * G * 64)
    put = fn(L, "requestToCreq", None, C.POINTER(Buf), C.POINTER(Buf), C.c_int32, C.c_int64, C.c_uint8, C.POINTER(Buf), C.c_int32,
             C.POINTER(Buf), C.c_int32, C.c_int32, C.c_int32)
    L.fake_reset()
    ic = cin.as_c()
    empty = np.zeros(1, np.int64)
    for q, t in zip(recs, terms_of):
        put(C.byref(buf_of_array(np.array([q], dtype=ingest.REQ_REC))), C.byref(buf_of_array(t if len(t) else empty)), int(q["row"]),
            now(int(q["row"])), 0, C.byref(buf_of_struct(ic)), G, C.byref(buf_of_struct(place2.c)), *place2.caps)
    assert L.fake_throws() == 0, L.fake_thrown_message()
    assert place2.requests().req.tobytes() == got.req.tobytes() and place2.requests().op_esc.tobytes() == got.op_esc.tobytes()
    put(C.byref(buf_of_array(np.array([recs[0]], dtype=ingest.REQ_REC))), C.byref(buf_of_array(empty)), int(recs[0]["row"]), now(0), 0,
        C.byref(buf_of_struct(ic)), G, C.byref(buf_of_struct(place2.c)), *place2.caps)
    assert L.fake_throws() == 1 and L.fake_thrown_class() == b"java/lang/IllegalArgumentException"
    L.fake_reset()
    reps = np.zeros(len(recs), dtype=ingest.BATCH_REC)
    n = fn(L, "coutboxToReplies", C.c_int32, C.POINTER(Buf), C.c_int32, C.c_int32, C.POINTER(Buf), C.POINTER(Buf), C.c_int32, C.POINTER(Buf))(
        C.byref(buf_of_struct(co.as_c())), G, 1, C.byref(buf_of_array(np.ascontiguousarray(recs))), C.byref(buf_of_array(prow)), len(recs),
        C.byref(buf_of_array(reps)))
    assert L.fake_throws() == 0 and reps[:n].tobytes() == rc.tobytes()

