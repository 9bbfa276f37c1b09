"""Host-side codec of the COMPACT host path (include/rafting_b200.h): what a transport shim does to the batches it exchanges
with the engine — numpy only.

  encode_inbox   dense lane events / group ops  ->  ev_c / op_c / row_base (+ escape records for whatever breaks a compact rule)
                 and, for steps with inbound requests, the request list (AppendEntries records + op escapes)
  decode_outbox  plan_c / rep_c / group columns / escape records  ->  the dense outbox columns

The engine's own unpack / pack kernels (rafting_b200/csrc/compact.cuh) are the inverse of these two; tests/test_compact_gpu.py
checks that a compact step, decoded, equals the dense step of the oracle bit for bit.
"""
from __future__ import annotations

import numpy as np

from . import abi

U64 = np.uint64


class CompactInbox:
    def __init__(self, rows, n, F):
        self.rows, self.n, self.F = rows, n, F
        self.row_base = np.zeros(rows, dtype=np.int64)
        self.op_c = np.zeros((rows, n), dtype=np.uint32)
        self.op_unavail = None                                # [rows, n] uint16 when some follower is unavailable
        self.ev_c = np.zeros((rows, n, F), dtype=np.uint32)
        self.esc = np.zeros(0, dtype=abi.CESC_IN)

    def nbytes(self):
        return self.row_base.nbytes + sum(a.nbytes for a in (self.op_c, self.op_unavail, self.ev_c) if a is not None) + self.esc.nbytes

    def as_c(self) -> abi.CInboxC:
        c = abi.CInboxC()
        c.rows, c.n_esc = self.rows, len(self.esc)
        c.row_base = self.row_base.ctypes.data
        c.op_c = None if self.op_c is None else self.op_c.ctypes.data
        c.op_unavail = None if self.op_unavail is None else self.op_unavail.ctypes.data
        c.ev_c = None if self.ev_c is None else self.ev_c.ctypes.data
        c.esc = self.esc.ctypes.data if len(self.esc) else None
        return c


class CompactRequests:
    """Inbound requests of a compact step (rafting_creqs_t): AppendEntries records, op escapes and the escapes' entry terms."""

    def __init__(self, req=None, op_esc=None, ent_terms=None):
        self.req = np.zeros(0, dtype=abi.CREQ) if req is None else req
        self.op_esc = np.zeros(0, dtype=abi.CESC_OP) if op_esc is None else op_esc
        self.ent_terms = np.zeros(0, dtype=np.int64) if ent_terms is None else ent_terms
        self.req_entries = int(((self.req["meta"] >> np.uint32(5)) & np.uint32(0x3F)).sum())

    def nbytes(self):
        return self.req.nbytes + self.op_esc.nbytes + self.ent_terms.nbytes

    def as_c(self) -> abi.CReqsC:
        c = abi.CReqsC()
        c.n_req, c.n_op_esc = len(self.req), len(self.op_esc)
        c.req = self.req.ctypes.data if len(self.req) else None
        c.op_esc = self.op_esc.ctypes.data if len(self.op_esc) else None
        c.ent_terms = self.ent_terms.ctypes.data if len(self.ent_terms) else None
        c.ent_count, c.req_entries = len(self.ent_terms), self.req_entries
        return c


class CompactOutbox:
    def __init__(self, rows, n, F, esc_cap=4096):
        self.rows, self.n, self.F, self.esc_cap = rows, n, F, esc_cap
        self.plan_c = np.zeros((rows, n, F), dtype=np.uint32)
        self.rep_c = np.zeros((rows, n), dtype=np.uint8)
        self.commit_index = np.zeros(n, dtype=np.int64)
        self.current_term = np.zeros(n, dtype=np.int64)
        self.role_word = np.zeros(n, dtype=np.uint32)
        self.incarnation = np.zeros(n, dtype=np.uint32)
        self.err_word = np.zeros(n, dtype=np.uint32)
        self.last_entry = np.zeros(n, dtype=abi.I64X2)
        self.epoch = np.zeros(n, dtype=abi.I64X2)
        self.esc = np.zeros(esc_cap, dtype=abi.CESC_OUT)
        self.counts = np.zeros(4, dtype=np.uint32)

    COLS = ("plan_c", "rep_c", "commit_index", "current_term", "role_word", "incarnation", "err_word", "last_entry", "epoch")

    def nbytes(self):
        return sum(getattr(self, c).nbytes for c in self.COLS) + 16

    def as_c(self) -> abi.COutboxC:
        c = abi.COutboxC()
        for name in self.COLS:
            setattr(c, name, getattr(self, name).ctypes.data)
        c.esc, c.esc_cap, c.counts = self.esc.ctypes.data, self.esc_cap, self.counts.ctypes.data
        return c

    def tags(self) -> np.ndarray:
        """tag of every plan, [rows, n, F] (abi.CTAG_NONE = none)"""
        return ((self.plan_c >> np.uint32(5)) & np.uint32(63)).astype(np.uint8)


def outbox_in_block(block: np.ndarray, out_off, rows: int, n: int, F: int, esc_cap: int) -> CompactOutbox:
    """A CompactOutbox whose columns are views into ONE (pinned) uint8 block laid out by Engine.compact_layout: the engine then
    brings a launch's whole outbox down with a single copy."""
    co = CompactOutbox.__new__(CompactOutbox)
    co.rows, co.n, co.F, co.esc_cap = rows, n, F, esc_cap
    spec = (("plan_c", np.uint32, (rows, n, F)), ("rep_c", np.uint8, (rows, n)), ("commit_index", np.int64, (n,)),
            ("current_term", np.int64, (n,)), ("role_word", np.uint32, (n,)), ("incarnation", np.uint32, (n,)), ("err_word", np.uint32, (n,)),
            ("last_entry", abi.I64X2, (n,)), ("epoch", abi.I64X2, (n,)), ("counts", np.uint32, (4,)), ("esc", abi.CESC_OUT, (esc_cap,)))
    for k, (name, dt, shape) in enumerate(spec):
        cnt = int(np.prod(shape))
        nbytes = cnt * np.dtype(dt).itemsize
        setattr(co, name, block[int(out_off[k]):int(out_off[k]) + nbytes].view(dt).reshape(shape))
    return co


def inbox_in_block(block: np.ndarray, in_off, ci: CompactInbox) -> CompactInbox:
    """Copies an encoded inbox into ONE (pinned) uint8 block laid out by Engine.compact_layout (n_esc_in = len(ci.esc)) and
    returns the CompactInbox whose columns are views into it: one copy up per launch."""
    out = CompactInbox.__new__(CompactInbox)
    out.rows, out.n, out.F = ci.rows, ci.n, ci.F
    for k, name in enumerate(("row_base", "op_c", "op_unavail", "ev_c", "esc")):
        a = getattr(ci, name)
        if a is None or (name == "esc" and len(a) == 0):
            setattr(out, name, None if name != "esc" else np.zeros(0, dtype=abi.CESC_IN))
            continue
        v = block[int(in_off[k]):int(in_off[k]) + a.nbytes].view(a.dtype).reshape(a.shape)
        v[...] = a
        setattr(out, name, v)
    return out


def _encode_requests(ib: abi.Inbox, ok: np.ndarray, base: np.ndarray) -> tuple[CompactRequests, np.ndarray]:
    """The request list of a dense inbox: every op other than a SUBMIT / TIMEOUT without a draw, in slot order.  Returns it
    and the mask of the slots it carries (op_c leaves them NONE)."""
    rows, n = ib.rows, ib.n
    draw = ib.op_nr["y"]
    listed = (ok != 0) & (((ok != abi.OP_SUBMIT) & (ok != abi.OP_TIMEOUT)) | (draw != 0))
    at = np.flatnonzero(listed.reshape(-1))
    if len(at) == 0:
        return CompactRequests(), listed
    meta = ib.op_meta.reshape(-1)[at]
    kind = (meta & U64(0xFF)).astype(np.int64)
    peer = ((meta >> U64(8)) & U64(0xFF)).astype(np.int64)
    count = ((meta >> U64(16)) & U64(0xFFFF)).astype(np.int64)
    ent = (meta >> U64(32)).astype(np.int64)
    now, dr = ib.op_nr["x"].reshape(-1)[at], draw.reshape(-1)[at]
    a, b = ib.op_ab["x"].reshape(-1)[at], ib.op_ab["y"].reshape(-1)[at]
    cc = ib.op_cd["x"].reshape(-1)[at] if ib.op_cd is not None else np.zeros(len(at), np.int64)
    d = ib.op_cd["y"].reshape(-1)[at] if ib.op_cd is not None else np.zeros(len(at), np.int64)
    e = ib.op_e.reshape(-1)[at] if ib.op_e is not None else (b.astype(np.uint64) + U64(1)).astype(np.int64)
    dt = now - base[at // n]
    in_pool = ent + count <= ib.ent_count
    wrap = lambda x: x.astype(np.uint64)                                        # int64 arithmetic modulo 2^64, as the engine's
    dterm = wrap(a) - wrap(cc)
    dcommit = (wrap(d) - wrap(b)).astype(np.int64)
    fits = ((kind == abi.OP_AE_REQUEST) & (dr == 0) & (wrap(e) == wrap(b) + U64(1)) & (dterm < U64(1 << 32)) &
            (dcommit >= -(1 << 31)) & (dcommit < (1 << 31)) & (dt >= 0) & (dt <= 0xFFFF) & (count <= 63) & (peer < 32) & in_pool)
    for k in np.flatnonzero(fits & (count > 0)):                               # every entry carries the request's term
        fits[k] = bool((ib.ent_terms[ent[k]:ent[k] + count[k]] == a[k]).all())
    req = np.zeros(int(fits.sum()), dtype=abi.CREQ)
    req["slot"] = at[fits]
    req["meta"] = (peer[fits] | (count[fits] << 5) | (dt[fits] << 16)).astype(np.uint32)
    req["term"], req["prev_index"] = a[fits], b[fits]
    req["d_prev_term"], req["d_commit"] = dterm[fits].astype(np.uint32), dcommit[fits].astype(np.int32)
    esc_k = np.flatnonzero(~fits)
    op_esc = np.zeros(len(esc_k), dtype=abi.CESC_OP)
    terms, pos = [], 0
    for j, k in enumerate(esc_k):
        off = 0xFFFFFFFF                                                        # out of the dense pool: out of this one too
        if in_pool[k]:
            off = pos
            terms.append(ib.ent_terms[ent[k]:ent[k] + count[k]]); pos += int(count[k])
        op_esc[j] = (at[k], off, int(meta[k]) & 0xFFFFFFFF, now[k], dr[k], a[k], b[k], cc[k], d[k], e[k])
    return CompactRequests(req, op_esc, np.concatenate(terms).astype(np.int64) if terms else None), listed


def encode_inbox(ib: abi.Inbox, tags: np.ndarray | None, sent_term: np.ndarray | None, sent_inc: np.ndarray | None = None) -> CompactInbox:
    """ib: dense host inbox (any group ops, any lane events).
    tags[r, i, f]: the tag the RPC this event answers was sent under (plan_c of the step that emitted it); None = no acks yet.
    sent_term[i] / sent_inc[i]: the term those RPCs carried and the incarnation of the role object that sent them (the group's
    current_term / incarnation columns of the step that planned them).  The incarnation is not on the wire — the engine keeps
    it with the echo pair under the tag — so a reply whose incarnation differs from sent_inc (a plan that was itself escaped)
    travels in full.
    Inbound requests, and SUBMIT / TIMEOUT ops with an explicit election-timeout draw, go to the request list `.reqs`
    (CompactRequests; None when the step has none: then it is a RAFTING_INBOX_NO_REQUESTS step)."""
    rows, n, F = ib.rows, ib.n, ib.F
    if ib.gids is not None:
        raise ValueError("the compact path is dense (no active list)")
    c = CompactInbox(rows, n, F)
    ek = (ib.ev_meta & U64(0xF)).astype(np.int64) if ib.ev_meta is not None else np.zeros((rows, n, F), np.int64)
    has_op = ib.op_meta is not None
    ok = (ib.op_meta & U64(0xFF)) if has_op else None
    # row base = the smallest time of the row
    big = np.iinfo(np.int64).max
    t_ev = np.where(ek != 0, ib.ev_tn["y"], big).reshape(rows, -1).min(axis=1) if ib.ev_meta is not None else np.full(rows, big)
    t_op = np.where(ok != 0, ib.op_nr["x"], big).min(axis=1) if has_op else np.full(rows, big)
    base = np.minimum(t_ev, t_op)
    base[base == big] = 0
    c.row_base[:] = base
    c.reqs = None
    if has_op:
        reqs, listed = _encode_requests(ib, ok, base)
        if listed.any():
            c.reqs = reqs
            ok = np.where(listed, U64(0), ok)
        dt = np.where(ok != 0, ib.op_nr["x"] - base[:, None], 0)
        if (dt < 0).any() or (dt > 0xFFFF).any():
            raise ValueError("a group op lies more than 65.535 s after its row's base time: use the dense path for this step")
        unav = ib.op_ab["x"].astype(np.uint64) if ib.op_ab is not None else np.zeros((rows, n), np.uint64)
        unav[listed] = 0
        if (unav > U64(0xFFFF)).any():
            raise ValueError("unavailable mask beyond 16 lanes")
        count = np.where(listed, U64(0), (ib.op_meta >> U64(16)) & U64(0xFFFF))
        if (count > U64(0xFFF)).any():
            raise ValueError("more than 4095 commands in one SUBMIT: use the dense path for this step")
        c.op_c[:] = (ok | (count << U64(4)) | (dt.astype(np.uint64) << U64(16))).astype(np.uint32)
        if (unav != 0).any():
            c.op_unavail = unav.astype(np.uint16)
    else:
        c.op_c = None
    if ib.ev_meta is None:
        c.ev_c = None
        return c
    em = ib.ev_meta
    outcome = (em >> U64(4)) & U64(3)
    is_ack = (ek == abi.EV_AE_ACK) | (ek == abi.EV_IS_ACK)
    dt = np.where(ek != 0, ib.ev_tn["y"] - base[:, None, None], 0)
    tg = tags if tags is not None else np.full((rows, n, F), abi.CTAG_NONE, np.uint8)
    term_ok = (ib.ev_tn["x"] == (sent_term[None, :, None] if sent_term is not None else 0))
    inc_ok = ((em >> U64(32)) == (sent_inc.astype(np.uint64)[None, :, None] if sent_inc is not None else U64(0)))
    fits = is_ack & (dt >= 0) & (dt <= 0xFFFF) & (tg < 32) & ((outcome != abi.OUT_OK) | term_ok) & inc_ok
    word = (em & U64(0x7F)) | (np.where(outcome == abi.OUT_OK, 1, 0).astype(np.uint64) << U64(7)) | (tg.astype(np.uint64) << U64(8)) | \
           (dt.astype(np.uint64) << U64(16))
    c.ev_c[:] = np.where(fits, word, np.where(ek != 0, U64(abi.CEV_ESCAPED), U64(0))).astype(np.uint32)
    esc_at = np.flatnonzero(((ek != 0) & ~fits).reshape(-1))
    if len(esc_at):
        c.esc = np.zeros(len(esc_at), dtype=abi.CESC_IN)
        c.esc["slot"] = esc_at
        c.esc["ev_meta"] = em.reshape(-1)[esc_at]
        c.esc["term"] = ib.ev_tn["x"].reshape(-1)[esc_at]; c.esc["now_ms"] = ib.ev_tn["y"].reshape(-1)[esc_at]
        c.esc["epoch_at_send"] = ib.ev_el["x"].reshape(-1)[esc_at]; c.esc["last_at_send"] = ib.ev_el["y"].reshape(-1)[esc_at]
    return c


def decode_outbox(co: CompactOutbox, G: int | None = None) -> abi.Outbox:
    """The dense outbox a compact step stands for (rep_term / ballots / escaped plans come from the escape list)."""
    rows, n, F = co.rows, co.n, co.F
    if int(co.counts[0]) > co.esc_cap:
        raise OverflowError("escape list overflow: fetch the dense outbox (rafting_step_fetch_dense)")
    o = abi.Outbox(rows, n, F, n if G is None else G)
    pc = co.plan_c.astype(np.uint64)
    kind = (pc & U64(7)).astype(np.int64)
    hb = (pc >> U64(3)) & U64(1)
    esc = ((pc >> U64(4)) & U64(1)) != 0
    cnt = ((pc >> U64(11)) & U64(63)).astype(np.int64)
    dprev = ((pc >> U64(17)) & U64(255)).astype(np.int64)
    dcommit = ((pc >> U64(25)) & U64(127)).astype(np.int64)
    # a compact plan was sent by the role object that holds the group at the end of the step
    o.plan_meta[:] = np.where(kind != 0, kind.astype(np.uint64) | (hb << U64(4)) | (cnt.astype(np.uint64) << U64(16)) |
                              (co.incarnation.astype(np.uint64)[None, :, None] << U64(32)), U64(0))
    last_x, term = co.last_entry["x"][None, :, None], co.current_term[None, :, None]
    commit, ep = co.commit_index[None, :, None], co.epoch
    ae, isn = (kind == abi.PLAN_AE) & ~esc, (kind == abi.PLAN_IS) & ~esc
    prev = last_x - dprev
    o.plan_pp["x"] = np.where(ae, prev, np.where(isn, ep["x"][None, :, None], 0))
    o.plan_pp["y"] = np.where(ae, term, np.where(isn, ep["y"][None, :, None], 0))
    o.plan_lc["x"] = np.where(ae, prev + cnt, np.where(isn, ep["x"][None, :, None], 0))
    o.plan_lc["y"] = np.where(ae | isn, commit - dcommit, 0)
    o.plan_epoch[:] = np.where(kind != 0, ep["x"][None, :, None], 0)
    rc = co.rep_c.astype(np.uint32)
    compact_rep = (rc >> np.uint32(7)) != 0                                   # a valid reply with the group's end-of-step term
    o.rep_meta[:] = ((rc & np.uint32(0x3F)) << np.uint32(8)) | np.where(compact_rep, np.uint32(1) | (((rc >> np.uint32(6)) & np.uint32(1)) << np.uint32(1)), np.uint32(0))
    o.rep_term[:] = np.where(compact_rep, co.current_term[None, :], 0)
    for name in ("commit_index", "current_term", "role_word", "incarnation", "err_word", "last_entry"):
        getattr(o, name)[:n] = getattr(co, name)
    for r in co.esc[:int(co.counts[0])]:
        k, slot = int(r["kind"]), int(r["slot"])
        if k == abi.CESC_PLAN:
            rr, rest = divmod(slot, n * F); i, f = divmod(rest, F)
            o.plan_meta[rr, i, f] = int(r["meta"]) & ~0xFF00                  # the full plan word of an escaped plan, minus the tag
            o.plan_pp[rr, i, f] = (r["a"], r["b"]); o.plan_lc[rr, i, f] = (r["c"], r["d"]); o.plan_epoch[rr, i, f] = r["e"]
        elif k == abi.CESC_BALLOT:
            rr, i = divmod(slot, n)
            o.ballot_meta[rr, i] = r["meta"]; o.ballot_term[rr, i] = r["a"]; o.ballot_last[rr, i] = (r["b"], r["c"])
        elif k == abi.CESC_REPLY:
            rr, i = divmod(slot, n)
            o.rep_meta[rr, i] = r["meta"]; o.rep_term[rr, i] = r["a"]
    return o
