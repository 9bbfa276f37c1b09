"""Host-side codec of the COMPACT host path (include/rafting_b200.h): what a transport shim does to the batches it exchanges
with the engine — numpy only.

  encode_inbox   dense lane events / group ops  ->  ev_c / op_c / row_base (+ escape records for whatever breaks a compact rule)
                 and, for steps with inbound requests, the request list (AppendEntries records + op escapes)
  decode_outbox  plan_c / rep_c / group columns / escape records  ->  the dense outbox columns
  encode_inbox(sweep=True) also carries the dense inbox's row_now as the sweep column of rafting_step_begin_compact_sweep

A step over an active list (gids, rafting_step_begin_compact_active) has every column sized by len(gids), by position: the
compact inbox and outbox carry the list, and the decoded outbox has the RAFTING_INBOX_COMPACT_GROUPS shape.

The engine's own unpack / pack kernels (rafting_b200/csrc/compact.cuh) are the inverse of these two; tests/test_compact_gpu.py
checks that a compact step, decoded, equals the dense step of the oracle bit for bit.
"""
from __future__ import annotations

import numpy as np

from . import abi

U64 = np.uint64


class CompactInbox:
    def __init__(self, rows, n, F, gids=None):
        self.rows, self.n, self.F = rows, n, F
        self.gids = None if gids is None else np.ascontiguousarray(gids, dtype=np.uint32)   # active list: position i is gids[i]
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
    def __init__(self, rows, n, F, esc_cap=4096, gids=None):
        self.rows, self.n, self.F, self.esc_cap = rows, n, F, esc_cap
        self.gids = None if gids is None else np.ascontiguousarray(gids, dtype=np.uint32)   # active list: position i is gids[i]
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

    def tags(self, rpc_only: bool = False) -> np.ndarray:
        """tag of every plan, [rows, n, F] (abi.CTAG_NONE = none).  rpc_only: CTAG_NONE on every lane that holds no AE / IS
        plan, so that every tag names an AppendEntries / InstallSnapshot in flight (what encode_inbox(elections=True) needs
        for acks: its escaped words free their tag).  A kind-7 word (abi.COMPACT_PREV_TERM) is an AppendEntries."""
        t = ((self.plan_c >> np.uint32(5)) & np.uint32(63)).astype(np.uint8)
        if rpc_only:
            k = self.plan_c & np.uint32(7)
            t[(k != abi.PLAN_AE) & (k != abi.PLAN_IS) & (k != abi.CPLAN_AE_PREV_TERM)] = abi.CTAG_NONE
        return t

    def ballot_tags(self) -> np.ndarray:
        """tag of every compact ballot lane of a step begun with abi.COMPACT_ELECTIONS, [rows, n, F]; CTAG_NONE on every other
        lane (an escaped ballot takes no tag, and a lane's AE / IS tag never answers a vote)"""
        t = ((self.plan_c >> np.uint32(5)) & np.uint32(63)).astype(np.uint8)
        k = self.plan_c & np.uint32(7)
        t[(k != abi.CPLAN_PREVOTE) & (k != abi.CPLAN_VOTE)] = abi.CTAG_NONE
        return t


def outbox_in_block(block: np.ndarray, out_off, rows: int, n: int, F: int, esc_cap: int, gids=None) -> CompactOutbox:
    """A CompactOutbox whose columns are views into ONE (pinned) uint8 block laid out by Engine.compact_layout: the engine then
    brings a launch's whole outbox down with a single copy.  gids: the active list of the steps it will serve (n = len(gids))."""
    co = CompactOutbox.__new__(CompactOutbox)
    co.rows, co.n, co.F, co.esc_cap = rows, n, F, esc_cap
    co.gids = None if gids is None else np.ascontiguousarray(gids, dtype=np.uint32)
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
    out.gids = getattr(ci, "gids", None)
    for k, name in enumerate(("row_base", "op_c", "op_unavail", "ev_c", "esc")):
        a = getattr(ci, name)
        if a is None or (name == "esc" and len(a) == 0):
            setattr(out, name, None if name != "esc" else np.zeros(0, dtype=abi.CESC_IN))
            continue
        v = block[int(in_off[k]):int(in_off[k]) + a.nbytes].view(a.dtype).reshape(a.shape)
        v[...] = a
        setattr(out, name, v)
    return out


def _encode_requests(ib: abi.Inbox, ok: np.ndarray, base: np.ndarray, elections: bool = False) -> tuple[CompactRequests, np.ndarray]:
    """The request list of a dense inbox: every op other than a SUBMIT / TIMEOUT without a draw, in slot order.  Returns it
    and the mask of the slots it carries (op_c leaves them NONE).  elections: PreVote / RequestVote become records too."""
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
    vk = np.zeros(len(at), np.int64)
    if elections:                                                              # a record stands for d = e = 0, no entries
        vk = np.where(kind == abi.OP_PREVOTE_REQ, abi.CREQ_VOTE_PRE, np.where(kind == abi.OP_VOTE_REQ, abi.CREQ_VOTE_RV, 0))
        e_ok = (e == 0) if ib.op_e is not None else np.ones(len(at), bool)
        fits |= ((vk != 0) & (dr == 0) & (count == 0) & (ent == 0) & (d == 0) & e_ok & (dterm < U64(1 << 32)) &
                 (dt >= 0) & (dt <= 0xFFFF) & (peer < 32))
    req = np.zeros(int(fits.sum()), dtype=abi.CREQ)
    req["slot"] = at[fits]
    req["meta"] = (peer[fits] | (count[fits] << 5) | (vk[fits] << 11) | (dt[fits] << 16)).astype(np.uint32)
    req["term"], req["prev_index"] = a[fits], b[fits]
    req["d_prev_term"], req["d_commit"] = dterm[fits].astype(np.uint32), np.where(vk[fits] != 0, 0, dcommit[fits]).astype(np.int32)
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


def sweep_column(ib: abi.Inbox) -> np.ndarray:
    """The sweep column of a compact step that stands for the dense inbox ib: its row_now (int64 [rows]; zeros without one)."""
    if ib.row_now is None:
        return np.zeros(ib.rows, dtype=np.int64)
    return np.ascontiguousarray(ib.row_now[:ib.rows], dtype=np.int64)


def due_inbox(ib: abi.Inbox, cap: int) -> abi.Inbox:
    """The dense inbox of a step begun with rafting_step_begin_compact_due: ib over the host's list ib.gids (positional, the
    COMPACT_GROUPS shape; ib.n may be 0) followed by `cap` empty tail positions, whose groups the device chooses.  Encode it
    with encode_inbox(..., sweep=True): every column and slot is then positional with n = len(ib.gids) + cap, and the compact
    inbox's gids stay the host's list.  After the wait, CompactOutbox.gids = gids followed by the tail (Engine.step_compact_due)."""
    out = abi.Inbox.__new__(abi.Inbox)
    out.__dict__.update(ib.__dict__)
    out.n = ib.n + cap
    out.gids = np.ascontiguousarray(ib.gids if ib.gids is not None else np.zeros(0, np.uint32), dtype=np.uint32)
    for name in ("op_meta", "op_nr", "op_ab", "op_cd", "op_e", "ev_meta", "ev_tn", "ev_el"):
        col = getattr(ib, name)
        if col is not None:
            pad = np.zeros((col.shape[0], cap) + col.shape[2:], dtype=col.dtype)
            setattr(out, name, np.ascontiguousarray(np.concatenate([col, pad], axis=1)))
    return out


def _without_sweep_row_ops(ib: abi.Inbox, on: np.ndarray) -> abi.Inbox:
    """ib with every group op of the sweep rows `on` removed: the step ignores them, and a request record there is refused."""
    out = abi.Inbox.__new__(abi.Inbox)
    out.__dict__.update(ib.__dict__)
    out.op_meta = ib.op_meta.copy()
    out.op_meta[on] = 0
    return out


def encode_inbox(ib: abi.Inbox, tags: np.ndarray | None, sent_term: np.ndarray | None, sent_inc: np.ndarray | None = None,
                 elections: bool = False, ballot_term: np.ndarray | None = None, ballot_inc: np.ndarray | None = None,
                 ballot_tags: np.ndarray | None = None, sweep: bool = False) -> CompactInbox:
    """ib: dense host inbox (any group ops, any lane events), over the whole shard or over an active list (ib.gids: the compact
    inbox then carries the list, and every array below is per position of THIS step; a pump maps what it kept from the step
    that planned by gid).
    tags[r, i, f]: the tag the RPC this event answers was sent under (plan_c of the step that emitted it); None = no acks yet.
    sent_term[i] / sent_inc[i]: the term those RPCs carried and the incarnation of the role object that sent them (the group's
    current_term / incarnation columns of the step that planned them).  The incarnation is not on the wire — the engine keeps
    it with the echo pair under the tag — so a reply whose incarnation differs from sent_inc (a plan that was itself escaped)
    travels in full.
    Inbound requests, and SUBMIT / TIMEOUT ops with an explicit election-timeout draw, go to the request list `.reqs`
    (CompactRequests; None when the step has none: then it is a RAFTING_INBOX_NO_REQUESTS step).
    elections: the inbox of a step begun with abi.COMPACT_ELECTIONS.  Vote replies become ev_c words, PreVote / RequestVote
    requests become records, and every escaped word carries the tag of the RPC it answers, which unpack frees: an ack's from
    tags, which must then name AE / IS plans in flight only (CompactOutbox.tags(rpc_only=True)), a vote reply's from
    ballot_tags[r, i, f] (CompactOutbox.ballot_tags() of the step that emitted the ballot; None = no compact ballot, every
    vote reply travels in full).  ballot_term[r, i] / ballot_inc[r, i]: the term and the asking incarnation of the ballot the
    vote replies in (r, i) answer (the decoded ballot columns of that step); a reply whose incarnation differs travels in
    full.
    sweep: the inbox of a step begun with rafting_step_begin_compact_sweep.  `.sweep` holds ib.row_now (sweep_column), and the
    group ops of the sweep rows are dropped: the step ignores them there, and a request record on a sweep row is refused.
    Off (the default), row_now is not encoded: the compact step has no sweep rows."""
    if sweep:
        col = sweep_column(ib)
        if ib.op_meta is not None and (col != 0).any():
            ib = _without_sweep_row_ops(ib, col != 0)
        c = encode_inbox(ib, tags, sent_term, sent_inc, elections, ballot_term, ballot_inc, ballot_tags)
        c.sweep = col
        return c
    rows, n, F = ib.rows, ib.n, ib.F
    c = CompactInbox(rows, n, F, gids=ib.gids)
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
        reqs, listed = _encode_requests(ib, ok, base, elections)
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
    escaped = U64(abi.CEV_ESCAPED)
    if elections:
        is_vote = (ek == abi.EV_PV_REPLY) | (ek == abi.EV_RV_REPLY)
        bt = (ballot_term if ballot_term is not None else np.zeros((rows, n), np.int64))[:, :, None].astype(np.uint64)
        binc = (ballot_inc if ballot_inc is not None else np.zeros((rows, n), np.uint64))[:, :, None].astype(np.uint64)
        rt = ib.ev_tn["x"].astype(np.uint64)
        is_ok = outcome == abi.OUT_OK
        cterm = np.where(is_ok, bt - rt, U64(0))                                 # modulo 2^64: a higher term wraps past 7
        # only a compact ballot lane's tag answers a vote: an AE / IS tag on the same lane belongs to a plan still in flight
        tb = ballot_tags if ballot_tags is not None else np.full((rows, n, F), abi.CTAG_NONE, np.uint8)
        vfits = (is_vote & (dt >= 0) & (dt <= 0xFFFF) & (tb < 32) & (np.where(is_ok, cterm < U64(8), rt == U64(0))) &
                ((em >> U64(32)) == binc))
        vword = (em & U64(0x7F)) | ((tb.astype(np.uint64) & U64(0x1F)) << U64(8)) | (np.where(vfits, cterm, U64(0)) << U64(13)) | \
                (dt.astype(np.uint64) << U64(16))
        word = np.where(is_vote, vword, word)
        fits = fits | vfits
        own = np.where(is_ack, tg, np.where(is_vote, tb, abi.CTAG_NONE)).astype(np.uint64)
        escaped = U64(abi.CEV_ESCAPED) | (own << U64(8))                      # the escaped event's RPC frees its tag
    c.ev_c[:] = np.where(fits, word, np.where(ek != 0, escaped, U64(0))).astype(np.uint32)
    esc_at = np.flatnonzero(((ek != 0) & ~fits).reshape(-1))
    if len(esc_at):
        c.esc = np.zeros(len(esc_at), dtype=abi.CESC_IN)
        c.esc["slot"] = esc_at
        c.esc["ev_meta"] = em.reshape(-1)[esc_at]
        c.esc["term"] = ib.ev_tn["x"].reshape(-1)[esc_at]; c.esc["now_ms"] = ib.ev_tn["y"].reshape(-1)[esc_at]
        c.esc["epoch_at_send"] = ib.ev_el["x"].reshape(-1)[esc_at]; c.esc["last_at_send"] = ib.ev_el["y"].reshape(-1)[esc_at]
    return c


def decode_outbox(co: CompactOutbox, G: int | None = None, elections: bool = False, prev_term: bool = False) -> abi.Outbox:
    """The dense outbox a compact step stands for (rep_term / ballots / escaped plans come from the escape list).
    elections: the step was begun with abi.COMPACT_ELECTIONS, so plan_c lanes of kind CPLAN_PREVOTE / CPLAN_VOTE are ballots.
    prev_term: the step was begun with abi.COMPACT_PREV_TERM, so a lane of kind CPLAN_AE_PREV_TERM is an AE plan whose
    prevLogTerm lies dterm below the group's term.
    An active outbox (co.gids) decodes to the RAFTING_INBOX_COMPACT_GROUPS shape: group columns [n] by position, and o.gids."""
    rows, n, F = co.rows, co.n, co.F
    if int(co.counts[0]) > co.esc_cap:
        raise OverflowError("escape list overflow: fetch the dense outbox (rafting_step_fetch_dense)")
    active = getattr(co, "gids", None)
    if active is not None and G is not None and G != n:
        raise ValueError("an active outbox has n group entries by position")
    o = abi.Outbox(rows, n, F, n if G is None else G)
    o.gids = active
    pc = co.plan_c.astype(np.uint64)
    kind = (pc & U64(7)).astype(np.int64)
    older = (kind == abi.CPLAN_AE_PREV_TERM) if prev_term else np.zeros(kind.shape, bool)
    kind = np.where(older, abi.PLAN_AE, kind)
    if elections and F:
        bk = kind[:, :, 0]                                                       # every lane of a compact ballot has the word
        pre, vote = bk == abi.CPLAN_PREVOTE, bk == abi.CPLAN_VOTE
        has = pre | vote
        o.ballot_meta[:] = np.where(has, np.where(pre, U64(abi.BALLOT_PREVOTE), U64(abi.BALLOT_VOTE)) |
                                    (co.incarnation.astype(np.uint64)[None, :] << U64(32)), U64(0))
        o.ballot_term[:] = np.where(has, co.current_term[None, :] + pre.astype(np.int64), 0)
        o.ballot_last["x"] = np.where(has, co.last_entry["x"][None, :], 0)
        o.ballot_last["y"] = np.where(has, co.last_entry["y"][None, :], 0)
        kind = np.where(kind >= abi.CPLAN_PREVOTE, 0, kind)
    hb = (pc >> U64(3)) & U64(1)
    esc = ((pc >> U64(4)) & U64(1)) != 0
    cnt = ((pc >> U64(11)) & U64(63)).astype(np.int64)
    dprev = ((pc >> U64(17)) & U64(255)).astype(np.int64)
    dcommit = np.where(older, (pc >> U64(28)) & U64(15), (pc >> U64(25)) & U64(127)).astype(np.int64)
    dterm = np.where(older, ((pc >> U64(25)) & U64(7)) + U64(1), U64(0)).astype(np.int64)
    # a compact plan was sent by the role object that holds the group at the end of the step
    o.plan_meta[:] = np.where(kind != 0, kind.astype(np.uint64) | (hb << U64(4)) | (cnt.astype(np.uint64) << U64(16)) |
                              (co.incarnation.astype(np.uint64)[None, :, None] << U64(32)), U64(0))
    last_x, term = co.last_entry["x"][None, :, None], co.current_term[None, :, None]
    commit, ep = co.commit_index[None, :, None], co.epoch
    ae, isn = (kind == abi.PLAN_AE) & ~esc, (kind == abi.PLAN_IS) & ~esc
    prev = last_x - dprev
    o.plan_pp["x"] = np.where(ae, prev, np.where(isn, ep["x"][None, :, None], 0))
    o.plan_pp["y"] = np.where(ae, term - dterm, np.where(isn, ep["y"][None, :, None], 0))
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


def ae_ranges(co: CompactOutbox) -> tuple[np.ndarray, np.ndarray, np.ndarray, np.ndarray]:
    """The AppendEntries ranges a compact outbox asks payloads for, as a pump decodes them for rafting_log_gather: plans of
    kind AE (1, or 7 under RAFTING_COMPACT_PREV_TERM, or an escaped AE) with entries, in lane-slot order (row * n + position)
    * F + lane.  -> (lane slots, gids, first indices, counts); rafting_log_gather_step_begin walks the same plans on the device."""
    w = co.plan_c.reshape(-1)
    kind, esc = w & 7, (w >> 4) & 1
    first = np.zeros(len(w), np.int64)
    count = np.where(esc == 0, (w >> 11) & 63, 0).astype(np.int64)
    ae = (esc == 0) & ((kind == 1) | (kind == abi.CPLAN_AE_PREV_TERM))
    pos = (np.arange(len(w)) // co.F) % co.n
    first[ae] = co.last_entry["x"][pos[ae]] - ((w[ae] >> 17) & 255) + 1
    rec = co.esc[:min(int(co.counts[0]), co.esc_cap)]
    rec = rec[(rec["kind"] == abi.CESC_PLAN) & (rec["slot"] < len(w))]
    ek = rec["meta"] & 0xF
    ec = (rec["meta"] >> 16) & 0xFFFF
    s = rec["slot"].astype(np.int64)
    ae[s] = ek == abi.PLAN_AE
    count[s] = ec.astype(np.int64)
    first[s] = rec["a"] + 1
    t = np.flatnonzero(ae & (count > 0))
    gids = pos[t] if co.gids is None else co.gids[pos[t]].astype(np.int64)
    return t, gids, first[t], count[t]
