"""ctypes binding of the transport framing library (include/rafting_ingest.h, rafting_b200/csrc/ingest.cpp): the reference's
EventCodec frame layout restated in C so that the pump thread can cut a receive buffer into frames and route them to group
ids.  Host only — no CUDA, no torch."""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import _build, abi

_LIB = None

ENQ, ACK, SYN, MW, PM, BATCH = 0x05, 0x06, 0x16, 0x95, 0x9E, 0x1A
MAX_HEAD, MAX_BODY = 128, 1 << 26

FRAME = np.dtype([("type", "u1"), ("has_sequence", "u1"), ("ending", "u1"), ("_pad", "u1"), ("sequence", "<i4"),
                  ("head_off", "<u4"), ("head_len", "<u4"), ("body_off", "<u4"), ("body_len", "<u4")])
BATCH_REC = np.dtype([("gid", "<u4"), ("kind", "u1"), ("lane", "u1"), ("flags", "u1"), ("row", "u1"), ("incarnation", "<u4"),
                      ("_pad", "<u4"), ("term", "<i8"), ("epoch_at_send", "<i8"), ("last_at_send", "<i8")])
ACK_REC = np.dtype([("gid", "<u4"), ("kind", "u1"), ("success", "u1"), ("_pad", "<u2"), ("sequence", "<i4"), ("frame", "<u4"),
                    ("term", "<i8")])
APPLY_REC = np.dtype([("gid", "<u4"), ("_pad", "<u4"), ("first", "<i8"), ("last", "<i8")])
REQ_REC = np.dtype([("gid", "<u4"), ("kind", "u1"), ("src_slot", "u1"), ("dst_slot", "u1"), ("row", "u1"), ("incarnation", "<u4"),
                    ("count", "<u4"), ("term", "<i8"), ("a", "<i8"), ("b", "<i8"), ("commit", "<i8"), ("epoch", "<i8"), ("last", "<i8")])
assert FRAME.itemsize == 24 and BATCH_REC.itemsize == 40 and ACK_REC.itemsize == 24 and REQ_REC.itemsize == 64


def lib():
    global _LIB
    if _LIB is None:
        L = C.CDLL(_build.build_ingest())
        L.rafting_frame_scan.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_uint32, C.POINTER(C.c_uint32),
                                         C.POINTER(C.c_size_t), C.POINTER(C.c_int)]
        L.rafting_frame_encode.restype = C.c_size_t
        L.rafting_frame_encode.argtypes = [C.c_void_p, C.c_size_t, C.c_uint8, C.c_int, C.c_int32, C.c_char_p, C.c_uint32,
                                           C.c_char_p, C.c_uint32, C.c_int]
        L.rafting_scope_parse.argtypes = [C.c_char_p, C.c_uint32, C.POINTER(C.c_uint32), C.POINTER(C.c_uint32)]
        L.rafting_ctxmap_create.argtypes = [C.POINTER(C.c_void_p)]
        L.rafting_ctxmap_destroy.argtypes = [C.c_void_p]
        L.rafting_ctxmap_put.argtypes = [C.c_void_p, C.c_char_p, C.c_uint32, C.c_uint32]
        L.rafting_ctxmap_get.argtypes = [C.c_void_p, C.c_char_p, C.c_uint32, C.POINTER(C.c_uint32)]
        L.rafting_batch_to_inbox.argtypes = [C.c_void_p, C.c_uint32, C.c_int64, C.POINTER(abi.InboxC), C.c_uint32, C.c_uint32,
                                             C.POINTER(C.c_uint32)]
        L.rafting_reply_body_encode.restype = C.c_size_t
        L.rafting_reply_body_encode.argtypes = [C.c_void_p, C.c_size_t, C.c_int64, C.c_int]
        L.rafting_reply_body_decode.argtypes = [C.c_char_p, C.c_size_t, C.POINTER(C.c_int64), C.POINTER(C.c_int)]
        L.rafting_ack_frame_decode.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(C.c_uint32), C.POINTER(C.c_uint32),
                                               C.POINTER(C.c_int32), C.POINTER(C.c_int64), C.POINTER(C.c_int)]
        L.rafting_dispatch_create.argtypes = [C.c_uint32, C.c_uint32, C.c_uint32, C.POINTER(C.c_void_p)]
        L.rafting_dispatch_destroy.argtypes = [C.c_void_p]
        L.rafting_outbox_to_requests.argtypes = [C.c_void_p, C.POINTER(abi.OutboxC), C.c_uint32, C.c_void_p, C.c_uint32,
                                                 C.POINTER(C.c_uint32), C.POINTER(C.c_uint32)]
        L.rafting_request_to_inbox.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_int64, C.c_int, C.POINTER(abi.InboxC),
                                               C.c_uint32, C.c_uint32, C.POINTER(C.c_uint32)]
        L.rafting_outbox_to_replies.argtypes = [C.POINTER(abi.OutboxC), C.c_uint32, C.c_uint32, C.c_void_p, C.c_void_p, C.c_uint32,
                                                C.c_void_p, C.POINTER(C.c_uint32)]
        L.rafting_request_to_creq.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_int64, C.c_int, C.POINTER(abi.CInboxC),
                                              C.c_uint32, C.POINTER(abi.CReqsC), C.c_uint32, C.c_uint32, C.c_uint32]
        L.rafting_request_to_creq_ex.argtypes = L.rafting_request_to_creq.argtypes + [C.c_uint32]
        L.rafting_coutbox_to_requests.argtypes = [C.c_void_p, C.POINTER(abi.COutboxC), C.c_uint32, C.c_uint32, C.c_void_p, C.c_void_p,
                                                  C.c_uint32, C.POINTER(C.c_uint32), C.POINTER(C.c_uint32)]
        L.rafting_coutbox_to_replies.argtypes = [C.POINTER(abi.COutboxC), C.c_uint32, C.c_uint32, C.c_void_p, C.c_void_p, C.c_uint32,
                                                 C.c_void_p, C.POINTER(C.c_uint32)]
        L.rafting_outbox_apply_ranges.argtypes = [C.POINTER(abi.OutboxC), C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_void_p,
                                                  C.c_uint32, C.POINTER(C.c_uint32)]
        L.rafting_pending_create.argtypes = [C.c_uint32, C.POINTER(C.c_void_p)]
        L.rafting_pending_destroy.argtypes = [C.c_void_p]
        L.rafting_pending_put.argtypes = [C.c_void_p, C.c_uint32, C.c_int32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32,
                                          C.c_int64, C.c_int64, C.c_int64]
        L.rafting_failures_to_cinbox.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_uint32, C.c_int64, C.c_uint32,
                                                 C.POINTER(abi.CInboxC), C.c_uint32, C.c_uint32, C.c_void_p, C.c_uint32, C.POINTER(C.c_uint32),
                                                 C.c_void_p, C.POINTER(C.c_uint32), C.POINTER(C.c_uint32)]
        L.rafting_failures_to_cinbox_ex.argtypes = L.rafting_failures_to_cinbox.argtypes + [C.c_uint32]
        L.rafting_pending_remove.argtypes = [C.c_void_p, C.c_uint32, C.c_int32]
        L.rafting_pending_size.restype = C.c_uint32
        L.rafting_pending_size.argtypes = [C.c_void_p]
        L.rafting_acks_to_cinbox.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_int64, C.c_uint32, C.POINTER(abi.CInboxC),
                                             C.c_uint32, C.c_uint32, C.c_void_p, C.c_uint32, C.POINTER(C.c_uint32), C.c_void_p,
                                             C.POINTER(C.c_uint32), C.POINTER(C.c_uint32)]
        L.rafting_acks_to_cinbox_ex.argtypes = L.rafting_acks_to_cinbox.argtypes + [C.c_uint32]
        L.rafting_builder_create.argtypes = [C.c_uint32, C.c_uint32, C.POINTER(C.c_void_p)]
        L.rafting_builder_destroy.argtypes = [C.c_void_p]
        L.rafting_builder_push_submit.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32]
        L.rafting_builder_push_request.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
        L.rafting_builder_push_reply.argtypes = [C.c_void_p, C.c_void_p]
        L.rafting_builder_clear_group.argtypes = [C.c_void_p, C.c_uint32]
        L.rafting_builder_pending.restype = C.c_uint32
        L.rafting_builder_pending.argtypes = [C.c_void_p]
        L.rafting_builder_build.argtypes = [C.c_void_p, C.c_int64, C.POINTER(abi.InboxC), C.c_uint32, C.POINTER(C.c_uint32), C.c_void_p,
                                            C.c_void_p, C.c_uint32, C.POINTER(C.c_uint32)]
        L.rafting_ack_frames_decode.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.POINTER(C.c_uint32)]
        _LIB = L
    return _LIB


def reply_body_encode(term: int, success: bool) -> bytes:
    """The Kryo bytes of RaftResponse(term, success) as the reference's Serialization.writeObject emits them (restated from
    kryo 4.0.2's format; include/rafting_ingest.h)."""
    buf = C.create_string_buffer(64)
    n = lib().rafting_reply_body_encode(buf, len(buf), term, 1 if success else 0)
    return buf.raw[:n]


def reply_body_decode(body: bytes):
    """-> (term, success) or None when the bytes are not exactly one RaftResponse."""
    t, ok = C.c_int64(), C.c_int()
    if lib().rafting_reply_body_decode(body, len(body), C.byref(t), C.byref(ok)) != 0:
        return None
    return t.value, bool(ok.value)


def encode(ftype: int, head: bytes, body: bytes = b"", sequence: int | None = None, ending: bool = False) -> bytes:
    buf = C.create_string_buffer(24 + len(head) + len(body))    # 17 bytes of framing at most (sequence + EOT)
    n = lib().rafting_frame_encode(buf, len(buf), ftype, 0 if sequence is None else 1, sequence or 0, head, len(head), body, len(body),
                                   1 if ending else 0)
    if n == 0:
        raise ValueError("frame does not fit / exceeds the codec limits")
    return buf.raw[:n]


def scan(data: bytes, cap: int = 1024):
    """-> (rc, frames (structured array), consumed bytes, transparent)"""
    out = np.zeros(cap, dtype=FRAME)
    n, used, tr = C.c_uint32(), C.c_size_t(), C.c_int()
    buf = np.frombuffer(data, dtype=np.uint8) if len(data) else np.zeros(1, np.uint8)
    rc = lib().rafting_frame_scan(buf.ctypes.data, len(data), out.ctypes.data, cap, C.byref(n), C.byref(used), C.byref(tr))
    return rc, out[:n.value], used.value, bool(tr.value)


def scope_parse(head: bytes):
    k, off = C.c_uint32(), C.c_uint32()
    rc = lib().rafting_scope_parse(head, len(head), C.byref(k), C.byref(off))
    if rc:
        raise ValueError("unknown context " + head.decode(errors="replace"))
    return k.value, head[off.value:]


class CtxMap:
    def __init__(self):
        self._h = C.c_void_p()
        lib().rafting_ctxmap_create(C.byref(self._h))

    def put(self, ctx: bytes, gid: int):
        lib().rafting_ctxmap_put(self._h, ctx, len(ctx), gid)

    def get(self, ctx: bytes):
        g = C.c_uint32()
        return g.value if lib().rafting_ctxmap_get(self._h, ctx, len(ctx), C.byref(g)) == 0 else None

    def __del__(self):
        try:
            lib().rafting_ctxmap_destroy(self._h)
        except Exception:
            pass


def ack_frame_decode(data: bytes, frame, ctxmap: "CtxMap"):
    """One scanned ACK frame -> (gid, event kind, sequence, term, success), or None (not an ACK / unknown scope or context /
    a body that is not one RaftResponse)."""
    buf = np.frombuffer(data, dtype=np.uint8)
    fr = np.array([frame], dtype=FRAME)
    gid, kind, seq, term, ok = C.c_uint32(), C.c_uint32(), C.c_int32(), C.c_int64(), C.c_int()
    if lib().rafting_ack_frame_decode(buf.ctypes.data, fr.ctypes.data, ctxmap._h, C.byref(gid), C.byref(kind), C.byref(seq),
                                      C.byref(term), C.byref(ok)) != 0:
        return None
    return gid.value, kind.value, seq.value, term.value, bool(ok.value)


def ack_frames_decode(data: bytes, frames: np.ndarray, ctxmap: "CtxMap") -> np.ndarray:
    """Every ACK frame of a scanned buffer that decodes -> one ACK_REC (its `frame` = index into `frames`)."""
    buf = np.frombuffer(data, dtype=np.uint8)
    frames = np.ascontiguousarray(frames, dtype=FRAME)
    out = np.zeros(max(1, len(frames)), dtype=ACK_REC)
    n = C.c_uint32()
    rc = lib().rafting_ack_frames_decode(buf.ctypes.data, frames.ctypes.data, len(frames), ctxmap._h, out.ctypes.data, C.byref(n))
    if rc:
        raise ValueError(f"rafting_ack_frames_decode: rc={rc}")
    return out[:n.value]


def batch_to_inbox(recs: np.ndarray, now_ms: int, inbox: abi.Inbox) -> tuple[int, int]:
    recs = np.ascontiguousarray(recs, dtype=BATCH_REC)
    done = C.c_uint32()
    ic = inbox.as_c()
    rc = lib().rafting_batch_to_inbox(recs.ctypes.data, len(recs), now_ms, C.byref(ic), inbox.n, inbox.F, C.byref(done))
    return rc, done.value


class Dispatch:
    """The pump's dispatch loop in C (include/rafting_ingest.h): host outbox -> request records; remembers the term of the
    role objects (incarnations) it has seen per group."""

    def __init__(self, n_groups: int, F: int, local_slot: int):
        self._h = C.c_void_p()
        rc = lib().rafting_dispatch_create(n_groups, F, local_slot, C.byref(self._h))
        if rc:
            raise ValueError(f"rafting_dispatch_create: rc={rc}")
        self.cap = 0

    def requests(self, outbox: abi.Outbox, rows: int, cap: int = 1 << 16):
        """-> (records, plans skipped because their role object's term is unknown)"""
        out = np.zeros(cap, dtype=REQ_REC)
        n, unk = C.c_uint32(), C.c_uint32()
        oc = outbox.as_c()
        rc = lib().rafting_outbox_to_requests(self._h, C.byref(oc), rows, out.ctypes.data, cap, C.byref(n), C.byref(unk))
        if rc:
            raise ValueError(f"rafting_outbox_to_requests: rc={rc}")
        return out[:n.value], unk.value

    def crequests(self, cout, rows: int, flags: int = 0, cap: int = 1 << 16):
        """The same from a waited-for compact outbox (rafting_b200.compact.CompactOutbox) of a step begun with `flags`
        -> (records, the tag of each record's pending entry, unknown plans); OverflowError when its escape list overflowed."""
        out = np.zeros(cap, dtype=REQ_REC)
        tags = np.zeros(cap, dtype=np.uint8)
        n, unk = C.c_uint32(), C.c_uint32()
        oc = cout.as_c()
        rc = lib().rafting_coutbox_to_requests(self._h, C.byref(oc), rows, flags, out.ctypes.data, tags.ctypes.data, cap, C.byref(n),
                                               C.byref(unk))
        if rc == -5 and int(cout.counts[0]) > cout.esc_cap:                    # RAFTING_E_CAPACITY
            raise OverflowError("escape list overflow: fetch the dense outbox (rafting_step_fetch_dense)")
        if rc:
            raise ValueError(f"rafting_coutbox_to_requests: rc={rc}")
        return out[:n.value], tags[:n.value], unk.value

    def __del__(self):
        try:
            lib().rafting_dispatch_destroy(self._h)
        except Exception:
            pass


def request_to_inbox(rec, entry_terms, row: int, now_ms: int, host_result: bool, inbox: abi.Inbox) -> int:
    """One request record -> the op slot (row, rec.gid) of a dense host inbox; returns the status code."""
    r = np.array([rec], dtype=REQ_REC)
    terms = np.ascontiguousarray(entry_terms, dtype=np.int64)
    ic = inbox.as_c()
    cnt = C.c_uint32(inbox.ent_count)
    rc = lib().rafting_request_to_inbox(r.ctypes.data, terms.ctypes.data if len(terms) else None, row, now_ms, 1 if host_result else 0,
                                        C.byref(ic), inbox.n, len(inbox.ent_terms), C.byref(cnt))
    if rc == 0:
        inbox.ent_count = cnt.value
    return rc


def outbox_to_replies(outbox: abi.Outbox, n_groups: int, local_slot: int, placed: np.ndarray, placed_row) -> np.ndarray:
    """The replies (BATCH_REC, for batch_to_inbox on the sender's side) to the request records placed in this step."""
    placed = np.ascontiguousarray(placed, dtype=REQ_REC)
    rows = np.ascontiguousarray(placed_row, dtype=np.uint8)
    out = np.zeros(max(1, len(placed)), dtype=BATCH_REC)
    n = C.c_uint32()
    oc = outbox.as_c()
    rc = lib().rafting_outbox_to_replies(C.byref(oc), n_groups, local_slot, placed.ctypes.data, rows.ctypes.data, len(placed),
                                         out.ctypes.data, C.byref(n))
    if rc:
        raise ValueError(f"rafting_outbox_to_replies: rc={rc}")
    return out[:n.value]


class CReqPlacer:
    """The request list of one compact step, filled by rafting_request_to_creq (the compact analogue of request_to_inbox)."""

    def __init__(self, req_cap: int, esc_cap: int, ent_cap: int):
        self.req = np.zeros(max(1, req_cap), dtype=abi.CREQ)
        self.op_esc = np.zeros(max(1, esc_cap), dtype=abi.CESC_OP)
        self.ent_terms = np.zeros(max(1, ent_cap), dtype=np.int64)
        self.caps = (req_cap, esc_cap, ent_cap)
        self.c = abi.CReqsC()
        self.c.req, self.c.op_esc, self.c.ent_terms = self.req.ctypes.data, self.op_esc.ctypes.data, self.ent_terms.ctypes.data

    def put(self, rec, entry_terms, row: int, now_ms: int, host_result: bool, cin, n_groups: int, flags: int = 0) -> int:
        """One request record -> a record or an op escape at (row, rec.gid) of the compact step `cin`; returns the status code.
        flags = abi.COMPACT_ELECTIONS: PreVote / RequestVote become vote records (rafting_request_to_creq_ex)."""
        r = np.array([rec], dtype=REQ_REC)
        terms = np.ascontiguousarray(entry_terms, dtype=np.int64)
        ic = cin.as_c()
        args = (r.ctypes.data, terms.ctypes.data if len(terms) else None, row, now_ms, 1 if host_result else 0, C.byref(ic), n_groups,
                C.byref(self.c), *self.caps)
        return lib().rafting_request_to_creq_ex(*args, flags) if flags else lib().rafting_request_to_creq(*args)

    def requests(self):
        """-> rafting_b200.compact.CompactRequests (copies of the lists placed so far)"""
        from .compact import CompactRequests
        c = self.c
        return CompactRequests(self.req[:c.n_req].copy(), self.op_esc[:c.n_op_esc].copy(), self.ent_terms[:c.ent_count].copy())


def coutbox_to_replies(cout, n_groups: int, local_slot: int, placed: np.ndarray, placed_row) -> np.ndarray:
    """outbox_to_replies over a compact outbox (rafting_b200.compact.CompactOutbox): replies from rep_c and the escape list."""
    placed = np.ascontiguousarray(placed, dtype=REQ_REC)
    rows = np.ascontiguousarray(placed_row, dtype=np.uint8)
    out = np.zeros(max(1, len(placed)), dtype=BATCH_REC)
    n = C.c_uint32()
    oc = cout.as_c()
    rc = lib().rafting_coutbox_to_replies(C.byref(oc), n_groups, local_slot, placed.ctypes.data, rows.ctypes.data, len(placed),
                                          out.ctypes.data, C.byref(n))
    if rc:
        raise ValueError(f"rafting_coutbox_to_replies: rc={rc}")
    return out[:n.value]


def apply_ranges(outbox: abi.Outbox, applied: np.ndarray, gids=None) -> np.ndarray:
    """Commit records of one step -> (gid, first, last) ranges to apply; advances `applied` (int64 per gid) in place."""
    assert applied.dtype == np.int64 and applied.flags.c_contiguous
    n = len(outbox.role_word) if gids is None else len(gids)
    g = None if gids is None else np.ascontiguousarray(gids, dtype=np.uint32)
    out = np.zeros(max(1, n), dtype=APPLY_REC)
    k = C.c_uint32()
    oc = outbox.as_c()
    rc = lib().rafting_outbox_apply_ranges(C.byref(oc), None if g is None else g.ctypes.data, n, applied.ctypes.data, len(applied),
                                           out.ctypes.data, len(out), C.byref(k))
    if rc:
        raise ValueError(f"rafting_outbox_apply_ranges: rc={rc}")
    return out[:k.value]


class Pending:
    """The pump's pending-invocation table: (peer, sequence) -> what the request was sent with (include/rafting_ingest.h)."""

    def __init__(self, capacity_hint: int = 0):
        self._h = C.c_void_p()
        rc = lib().rafting_pending_create(capacity_hint, C.byref(self._h))
        if rc:
            raise ValueError(f"rafting_pending_create: rc={rc}")

    def put(self, peer, sequence, ev_kind, gid, lane, tag, incarnation, term, epoch_at_send, last_at_send):
        rc = lib().rafting_pending_put(self._h, peer, sequence, ev_kind, gid, lane, tag, incarnation, term, epoch_at_send, last_at_send)
        if rc:
            raise ValueError(f"rafting_pending_put: rc={rc}")

    def remove(self, peer, sequence) -> bool:
        return lib().rafting_pending_remove(self._h, peer, sequence) == 0

    def __len__(self):
        return lib().rafting_pending_size(self._h)

    def acks_to_cinbox(self, peer: int, acks: np.ndarray, now_ms: int, row: int, cin, esc: np.ndarray, n_esc: int, flags: int = 0):
        """Writes the replies into row `row` of the compact inbox `cin` (rafting_b200.compact.CompactInbox with ev_c allocated);
        -> (status, escape records used so far, indices of deferred acks, unknown sequences).  flags = abi.COMPACT_ELECTIONS:
        vote replies become vote words and escaped words carry their tag (rafting_acks_to_cinbox_ex)."""
        acks = np.ascontiguousarray(acks, dtype=ACK_REC)
        deferred = np.zeros(max(1, len(acks)), dtype=np.uint32)
        ne, nd, nu = C.c_uint32(n_esc), C.c_uint32(), C.c_uint32()
        cc = cin.as_c()
        args = (self._h, peer, acks.ctypes.data, len(acks), now_ms, row, C.byref(cc), cin.n, cin.F, esc.ctypes.data, len(esc), C.byref(ne),
                deferred.ctypes.data, C.byref(nd), C.byref(nu))
        rc = lib().rafting_acks_to_cinbox_ex(*args, flags) if flags else lib().rafting_acks_to_cinbox(*args)
        return rc, ne.value, deferred[:nd.value].copy(), nu.value

    def failures_to_cinbox(self, peer: int, sequences, outcome: int, now_ms: int, row: int, cin, esc: np.ndarray, n_esc: int,
                           flags: int = 0):
        """Invocations that timed out (OUT_ERROR) / were cancelled (OUT_CANCELED): same contract as acks_to_cinbox."""
        seqs = np.ascontiguousarray(sequences, dtype=np.int32)
        deferred = np.zeros(max(1, len(seqs)), dtype=np.uint32)
        ne, nd, nu = C.c_uint32(n_esc), C.c_uint32(), C.c_uint32()
        cc = cin.as_c()
        args = (self._h, peer, seqs.ctypes.data, len(seqs), outcome, now_ms, row, C.byref(cc), cin.n, cin.F, esc.ctypes.data, len(esc),
                C.byref(ne), deferred.ctypes.data, C.byref(nd), C.byref(nu))
        rc = lib().rafting_failures_to_cinbox_ex(*args, flags) if flags else lib().rafting_failures_to_cinbox(*args)
        return rc, ne.value, deferred[:nd.value].copy(), nu.value

    def __del__(self):
        try:
            lib().rafting_pending_destroy(self._h)
        except Exception:
            pass


class Builder:
    """Per-group FIFOs of requests / replies / submits -> the rows of one dense step (include/rafting_ingest.h)."""

    def __init__(self, n_groups: int, F: int):
        self._h = C.c_void_p()
        rc = lib().rafting_builder_create(n_groups, F, C.byref(self._h))
        if rc:
            raise ValueError(f"rafting_builder_create: rc={rc}")
        self.G, self.F = n_groups, F

    def push_submit(self, gid, count, unavailable_mask=0):
        rc = lib().rafting_builder_push_submit(self._h, gid, count, unavailable_mask)
        if rc:
            raise ValueError(f"rafting_builder_push_submit: rc={rc}")

    def push_request(self, rec, entry_terms=()):
        r = np.array([rec], dtype=REQ_REC)
        t = np.ascontiguousarray(entry_terms, dtype=np.int64)
        rc = lib().rafting_builder_push_request(self._h, r.ctypes.data, t.ctypes.data if len(t) else None)
        if rc:
            raise ValueError(f"rafting_builder_push_request: rc={rc}")

    def push_reply(self, rec):
        r = np.array([rec], dtype=BATCH_REC)
        rc = lib().rafting_builder_push_reply(self._h, r.ctypes.data)
        if rc:
            raise ValueError(f"rafting_builder_push_reply: rc={rc}")

    def clear_group(self, gid):
        lib().rafting_builder_clear_group(self._h, gid)

    def __len__(self):
        return lib().rafting_builder_pending(self._h)

    def build(self, now_ms: int, inbox: abi.Inbox, placed_cap: int = 4096):
        """Fills `inbox` (dense, sweep row, every column allocated); -> (placed records, their rows)."""
        placed = np.zeros(placed_cap, dtype=REQ_REC)
        rows = np.zeros(placed_cap, dtype=np.uint8)
        ic = inbox.as_c()
        cnt, n = C.c_uint32(), C.c_uint32()
        rc = lib().rafting_builder_build(self._h, now_ms, C.byref(ic), len(inbox.ent_terms), C.byref(cnt), placed.ctypes.data,
                                         rows.ctypes.data, placed_cap, C.byref(n))
        if rc:
            raise ValueError(f"rafting_builder_build: rc={rc}")
        inbox.ent_count = cnt.value
        return placed[:n.value], rows[:n.value]

    def __del__(self):
        try:
            lib().rafting_builder_destroy(self._h)
        except Exception:
            pass
