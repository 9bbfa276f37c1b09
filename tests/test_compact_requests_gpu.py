"""Inbound requests through the compact host path (`-m gpu`): a config #5 step fed through rafting_step_begin_compact_req
(AppendEntries as 32-byte records, every other request as an op escape, replies in rep_c) must be, once decoded, bit for bit
the dense step of the oracle on the same logical stream, in the class-sorted launch (G >= 2048) and the unsorted one.
Malformed request lists are answered per op with RAFTING_ERR_BAD_EVENT, exactly as the oracle answers the equivalent dense
inbox, and an escape-list overflow falls back losslessly to the dense outbox."""
import numpy as np
import pytest

from oracle import binding
from rafting_b200 import abi, compact, workload
from tests import harness

pytestmark = pytest.mark.gpu
U64 = np.uint64
SEED = 0x5EED0005


def _pair(G, R, rows, pool=None):
    from rafting_b200 import engine
    cfg = abi.make_cfg(replicas=R, max_groups=G, max_rows=rows, entry_pool_cap=rows * G * 50 if pool is None else pool)
    e, o = engine.Engine(cfg), binding.Oracle(cfg)
    init = harness.init_array(G, terms=np.arange(G) % 7)
    e.open_bulk(0, init), o.open_bulk(0, init)
    w1 = workload.make_wl(SEED, 1, G, R - 1)
    harness.assert_outbox_equal(harness.elect_all(o, w1), harness.elect_all(e, w1), where="election (dense path)")
    return e, o


def _run_mixed(G, R, rows, steps, settle=8):
    e, o = _pair(G, R, rows)
    F = R - 1
    w = workload.make_wl(SEED, rows, G, F)
    prev, tags, sent_term, sent_inc = None, None, None, None
    ae = records = valid = compact_replies = 0
    for k in range(steps):
        ib = workload.mixed_inbox_host(w, k, prev)
        want = o.step(ib, threads=8)
        cin = compact.encode_inbox(ib, tags, sent_term, sent_inc)
        reqs = cin.reqs if cin.reqs is not None else compact.CompactRequests()
        cout = compact.CompactOutbox(rows, G, F, esc_cap=rows * G * F + 2 * rows * G)     # room for every record: no fallback
        e.step_compact(cin, cout, reqs=reqs)
        harness.assert_outbox_equal(want, compact.decode_outbox(cout), where=f"compact step {k}")
        if k >= settle:
            ae += int(((ib.op_meta & U64(0xFF)) == abi.OP_AE_REQUEST).sum())
            records += len(reqs.req)
            valid += int((want.rep_meta & 1).sum())
            compact_replies += int((cout.rep_c >> 7).sum())
        prev, tags, sent_term, sent_inc = want, cout.tags(), cout.current_term.copy(), cout.incarnation.copy()
    harness.assert_states_equal(o, e, list(range(0, G, max(1, G // 97))) + [G - 1], F, where="compact requests end")
    assert ae > 0 and valid > 0
    assert records >= 0.9 * ae, (records, ae)
    assert compact_replies >= 0.9 * valid, (compact_replies, valid)


def test_config5_through_the_request_list_class_sorted_launch():
    _run_mixed(G=16384, R=3, rows=4, steps=40)


def test_config5_through_the_request_list_unsorted_launch():
    _run_mixed(G=1024, R=5, rows=4, steps=40)


def _malformed(ib: abi.Inbox, r: int, i: int, row_base):
    ib.op_meta[r, i] = abi.COP_MALFORMED
    ib.op_nr[r, i] = (row_base[r], 0)
    ib.op_ab[r, i] = (0, 0); ib.op_cd[r, i] = (0, 0); ib.op_e[r, i] = 0


def test_malformed_request_lists_are_answered_per_op_like_the_dense_step():
    from rafting_b200 import engine
    G, R, rows = 1024, 3, 4
    F = R - 1
    e, o = _pair(G, R, rows)
    w = workload.make_wl(SEED, rows, G, F)
    prev = None
    for k in range(10):                                           # dense steps until followers receive entries
        ib = workload.mixed_inbox_host(w, k, prev)
        prev = o.step(ib)
        harness.assert_outbox_equal(prev, e.step(ib), where=f"dense step {k}")
    ib = workload.mixed_inbox_host(w, 10, prev)
    cin = compact.encode_inbox(ib, None, None, None)
    q = cin.reqs
    req = q.req
    cnt = (req["meta"] >> np.uint32(5)) & np.uint32(0x3F)
    last = int(np.flatnonzero(cnt > 0)[-1])                       # understated req_entries: this record's terms fall off the pool
    dup = 0                                                        # the same slot twice in the record list
    assert dup < last
    sub = np.argwhere((cin.op_c & np.uint32(0xF)) == abi.OP_SUBMIT)[0]
    s_sub = int(sub[0]) * G + int(sub[1])                          # a record on a slot that already has an op_c word
    extra = np.zeros(1, dtype=abi.CREQ)
    extra["slot"], extra["meta"], extra["term"], extra["prev_index"] = s_sub, abi.creq_make(1, 0, 0), 5, 3
    bad_req = np.sort(np.concatenate([req[:dup + 1], req[dup:], extra]), order="slot", kind="stable")
    reqs = compact.CompactRequests(bad_req, q.op_esc, q.ent_terms)
    reqs.req_entries -= 1
    # the equivalent dense inbox: an unknown op kind on the claimed slots, an out-of-pool entry offset on the last record
    want_ib = ib
    for s in (int(req[dup]["slot"]), s_sub):
        _malformed(want_ib, s // G, s % G, cin.row_base)
    s_last = int(req[last]["slot"])
    want_ib.op_meta[s_last // G, s_last % G] = (want_ib.op_meta[s_last // G, s_last % G] & U64(0xFFFFFFFF)) | (U64(want_ib.ent_count) << U64(32))
    want = o.step(want_ib)
    cout = compact.CompactOutbox(rows, G, F, esc_cap=rows * G * F + 2 * rows * G)
    e.step_compact(cin, cout, reqs=reqs)
    got = compact.decode_outbox(cout)
    harness.assert_outbox_equal(want, got, where="malformed request list")
    for s in (int(req[dup]["slot"]), s_sub, s_last):
        assert (int(got.rep_meta[s // G, s % G]) >> 8) == abi.ERR["BAD_EVENT"]
    harness.assert_states_equal(o, e, range(0, G, 7), F, where="after the malformed step")
    # an entry pool larger than the engine's: refused at call level
    over = compact.CompactRequests(q.req, q.op_esc, q.ent_terms)
    over.req_entries = e.cfg.entry_pool_cap - len(q.ent_terms) + 1
    with pytest.raises(engine.RaftingError) as ex:
        e.step_compact(cin, compact.CompactOutbox(rows, G, F), reqs=over)
    assert ex.value.rc == -5


def test_escape_overflow_with_requests_falls_back_to_the_dense_outbox():
    G, R, rows = 1024, 3, 4
    F = R - 1
    e, o = _pair(G, R, rows)
    w = workload.make_wl(SEED, rows, G, F)
    ib = workload.mixed_inbox_host(w, 0, None)
    prev = o.step(ib)
    harness.assert_outbox_equal(prev, e.step(ib), where="dense step 0")
    ib = workload.mixed_inbox_host(w, 1, prev)                    # the stepped-down churn leaders' first AppendEntries
    want = o.step(ib)
    cin = compact.encode_inbox(ib, None, None, None)
    assert cin.reqs is not None and len(cin.reqs.req)
    cout = compact.CompactOutbox(rows, G, F, esc_cap=8)
    e.step_compact(cin, cout, reqs=cin.reqs)
    assert int(cout.counts[0]) > 8
    with pytest.raises(OverflowError):
        compact.decode_outbox(cout)
    dense = abi.Outbox(rows, G, F, G)
    e.step_fetch_dense(0, dense.as_c())
    harness.assert_outbox_equal(want, dense, where="dense fallback")


def test_step_begin_compact_req_through_the_jni_glue(tmp_path):
    """stepBeginCompactReq / stepWaitCompact through the stand-in JNIEnv, in lock-step with the oracle."""
    import ctypes as C
    from tests import jni_exec
    from tests.jni_exec import Buf, buf_of_struct, fn
    L = jni_exec.build(str(tmp_path))
    if L is None:
        pytest.skip("no gcc")
    G, R, rows = 1024, 3, 4
    F = R - 1
    cfg = abi.make_cfg(replicas=R, max_groups=G, max_rows=rows, entry_pool_cap=rows * G * 50)
    o = binding.Oracle(cfg)
    L.fake_reset()
    h = fn(L, "create", C.c_int64, C.POINTER(Buf))(C.byref(buf_of_struct(cfg)))
    assert h != 0 and L.fake_throws() == 0, L.fake_thrown_message()
    init = harness.init_array(G, terms=np.arange(G) % 7)
    o.open_bulk(0, init)
    fn(L, "groupOpenBulk", None, C.c_int64, C.c_int32, C.c_int32, C.POINTER(Buf))(h, 0, G, C.byref(jni_exec.buf_of_array(init)))
    begin_host = fn(L, "stepBeginHost", None, C.c_int64, C.c_int32, C.POINTER(Buf), C.POINTER(Buf))
    wait_slot = fn(L, "stepWaitSlot", None, C.c_int64, C.c_int32)
    begin = fn(L, "stepBeginCompactReq", None, C.c_int64, C.c_int32, C.POINTER(Buf), C.POINTER(Buf), C.POINTER(Buf))
    wait = fn(L, "stepWaitCompact", None, C.c_int64, C.c_int32)
    w1 = workload.make_wl(SEED, 1, G, F)
    prev = None
    for ph in (0, 1, 2):                                          # the election through the dense natives
        ib = workload.election_inbox_host(w1, ph, prev)
        prev = o.step(ib)
        out = abi.Outbox(1, G, F, G)
        begin_host(h, 0, C.byref(buf_of_struct(ib.as_c())), C.byref(buf_of_struct(out.as_c()))); wait_slot(h, 0)
        harness.assert_outbox_equal(prev, out, where=f"election phase {ph}")
    w = workload.make_wl(SEED, rows, G, F)
    prev, tags, sent_term, sent_inc, with_requests = None, None, None, None, 0
    for k in range(12):
        ib = workload.mixed_inbox_host(w, k, prev)
        want = o.step(ib)
        cin = compact.encode_inbox(ib, tags, sent_term, sent_inc)
        reqs = cin.reqs if cin.reqs is not None else compact.CompactRequests()
        with_requests += len(reqs.req) > 0
        cout = compact.CompactOutbox(rows, G, F, esc_cap=rows * G * F + 2 * rows * G)
        begin(h, k % 4, C.byref(buf_of_struct(cin.as_c())), C.byref(buf_of_struct(reqs.as_c())), C.byref(buf_of_struct(cout.as_c())))
        wait(h, k % 4)
        assert L.fake_throws() == 0, L.fake_thrown_message()
        harness.assert_outbox_equal(want, compact.decode_outbox(cout), where=f"compact step {k} through the natives")
        prev, tags, sent_term, sent_inc = want, cout.tags(), cout.current_term.copy(), cout.incarnation.copy()
    assert with_requests > 0
    fn(L, "destroy", None, C.c_int64)(h)
