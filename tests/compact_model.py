"""numpy restatement of the engine's compact kernels (rafting_b200/csrc/compact.cuh) and the host side of a compact pump
around it — TEST INFRASTRUCTURE.

  pack / unpack      pack_kernel<EL, PT>, and unpack_kernel<EL> + unpack_escapes_kernel + unpack_requests_kernel<EL>, keyed by
                     the step's flags word (abi.COMPACT_ELECTIONS = EL, abi.COMPACT_PREV_TERM = PT) as the kernels are
  prev_term_words    the only restatement of the kind-7 rule: what PT changes in a packed outbox
  encode / next_of   what a pump encodes a step's inbox with, and what it keeps from the step for the next one
  Driver             such a pump around the engine, checked against the oracle every step (-m gpu)

The CPU suites (tests/test_compact_*_cpu.py) run the model around the oracle to check that the compact wire format of
include/rafting_b200.h is lossless without a GPU; under -m gpu the real kernels are checked against the oracle and the
model (tests/test_compact_*_gpu.py)."""
from __future__ import annotations

import numpy as np

from oracle import binding
from rafting_b200 import abi, compact, workload
from tests import harness

CTAGS = 32
U64 = np.uint64
M64 = (1 << 64) - 1
EL, PT = abi.COMPACT_ELECTIONS, abi.COMPACT_PREV_TERM


class InFlight:
    """The HBM in-flight table: per (group, follower) 32 tags -> (epochAtSend, lastIndexAtSend, incarnation) + a tag bitmap."""

    def __init__(self, G, F):
        self.el = np.zeros((CTAGS, G, F), dtype=abi.I64X2)
        self.inc = np.zeros((CTAGS, G, F), dtype=np.uint32)
        self.bits = np.zeros((G, F), dtype=np.uint32)


def ballot_lane_kind(dense: abi.Outbox, r: int, g: int) -> int:
    """The plan_c kind the ballot of (r, g) travels as under EL (CPLAN_PREVOTE / CPLAN_VOTE), or 0 when it stays an escape
    record."""
    bm = int(dense.ballot_meta[r, g])
    bk = bm & 0xFFFFFFFF
    if bk not in (abi.BALLOT_PREVOTE, abi.BALLOT_VOTE) or (bm >> 32) != int(dense.incarnation[g]):
        return 0
    pre = bk == abi.BALLOT_PREVOTE
    bl = dense.ballot_last[r, g]
    if (int(dense.ballot_term[r, g]) - int(dense.current_term[g])) & M64 != (1 if pre else 0):
        return 0
    if (int(bl["x"]), int(bl["y"])) != (int(dense.last_entry[g]["x"]), int(dense.last_entry[g]["y"])):
        return 0
    if (dense.plan_meta[r, g] != 0).any():
        return 0
    return abi.CPLAN_PREVOTE if pre else abi.CPLAN_VOTE


def _take(b: int) -> tuple[int, int]:
    free = ~b & 0xFFFFFFFF
    if not free:
        return abi.CTAG_NONE, b
    tag = (free & -free).bit_length() - 1
    return tag, b | (1 << tag)


def pack(dense: abi.Outbox, epoch: np.ndarray, st: InFlight, esc_cap: int, flags: int = 0,
         replies: bool = False) -> compact.CompactOutbox:
    """pack_kernel<EL, PT>: dense outbox -> compact outbox; tags handed out per lane in row order, lowest free first.
    replies (COutD.compact_replies: the step was begun with a request list): a valid reply whose term is the group's
    end-of-step term travels in rep_c (bit 7, success in bit 6) instead of the escape list.
    EL: a ballot that matches the end-of-step columns becomes one plan_c word per lane, each taking the lowest free tag of
    its lane, interleaved in row order with the AE / IS plans of the same lane.
    PT: every plan record that fits kind 7 becomes its word again (prev_term_words)."""
    el = bool(flags & EL)
    rows, n, F = dense.rows, dense.n, dense.F
    co = compact.CompactOutbox(rows, n, F, esc_cap=rows * n * F + 2 * rows * n if flags & PT else esc_cap)   # PT: every record
    for name in ("commit_index", "current_term", "role_word", "incarnation", "err_word", "last_entry"):
        getattr(co, name)[:] = getattr(dense, name)[:n]
    co.epoch[:] = epoch
    esc = []
    bkind = np.array([[ballot_lane_kind(dense, r, g) for g in range(n)] for r in range(rows)], np.int64).reshape(rows, n)
    for g in range(n):
        commit_end, term_end, inc_end = int(dense.commit_index[g]), int(dense.current_term[g]), int(dense.incarnation[g])
        last_end, ep = int(dense.last_entry[g]["x"]), (int(epoch[g]["x"]), int(epoch[g]["y"]))
        for f in range(F):
            b = int(st.bits[g, f])
            for r in range(rows):
                pm = int(dense.plan_meta[r, g, f])
                if pm == 0:
                    if el and bkind[r, g]:
                        tag, b = _take(b)
                        if tag != abi.CTAG_NONE:
                            st.el[tag, g, f] = (int(dense.ballot_term[r, g]), 0); st.inc[tag, g, f] = inc_end
                        co.plan_c[r, g, f] = int(bkind[r, g]) | (tag << 5)
                    continue
                kind, hb, count, inc = pm & 0xF, (pm >> 4) & 1, (pm >> 16) & 0xFFFF, pm >> 32
                pp, lc, pe = dense.plan_pp[r, g, f], dense.plan_lc[r, g, f], int(dense.plan_epoch[r, g, f])
                tag = abi.CTAG_NONE
                if kind in (abi.PLAN_AE, abi.PLAN_IS):
                    tag, b = _take(b)
                    if tag != abi.CTAG_NONE:
                        st.el[tag, g, f] = (pe, int(lc["x"])); st.inc[tag, g, f] = inc
                dcommit = (commit_end - int(lc["y"])) & M64
                dprev = 0
                fits = pe == ep[0] and inc == inc_end and count < 64
                if kind == abi.PLAN_AE:
                    dprev = (last_end - int(pp["x"])) & M64
                    fits = fits and int(pp["y"]) == term_end and int(lc["x"]) == int(pp["x"]) + count and dprev < 256 and dcommit < 128
                elif kind == abi.PLAN_IS:
                    fits = fits and (int(pp["x"]), int(pp["y"])) == ep and int(lc["x"]) == ep[0] and dcommit < 128
                else:
                    fits = fits and int(pp["x"]) == 0 and int(pp["y"]) == 0 and int(lc["x"]) == 0 and int(lc["y"]) == 0
                pc = kind | (hb << 3) | (tag << 5)
                if fits:
                    pc |= (count << 11) | (dprev << 17) | ((dcommit << 25) if kind in (abi.PLAN_AE, abi.PLAN_IS) else 0)
                else:
                    pc |= 1 << 4
                    esc.append((abi.CESC_PLAN, (r * n + g) * F + f, pm | ((255 if tag == abi.CTAG_NONE else tag) << 8),
                                int(pp["x"]), int(pp["y"]), int(lc["x"]), int(lc["y"]), pe))
                co.plan_c[r, g, f] = pc
            st.bits[g, f] = b
        for r in range(rows):
            rm = int(dense.rep_meta[r, g])
            co.rep_c[r, g] = (rm >> 8) & 0xFF
            if rm & 1:
                co.counts[2] += 1
                if replies and int(dense.rep_term[r, g]) == term_end:
                    co.rep_c[r, g] |= 0x80 | (((rm >> 1) & 1) << 6)
                else:
                    esc.append((abi.CESC_REPLY, r * n + g, rm, int(dense.rep_term[r, g]), 0, 0, 0, 0))
            bm = int(dense.ballot_meta[r, g])
            if bm:
                co.counts[1] += 1
                if not (el and bkind[r, g]):
                    bl = dense.ballot_last[r, g]
                    esc.append((abi.CESC_BALLOT, r * n + g, bm, int(dense.ballot_term[r, g]), int(bl["x"]), int(bl["y"]), 0, 0))
    co.counts[0] = len(esc)
    for k, rec in enumerate(esc[:co.esc_cap]):
        co.esc[k] = rec
    return prev_term_words(co, esc_cap) if flags & PT else co


def prev_term_word(co: compact.CompactOutbox, rec) -> int:
    """The kind-7 word an escaped plan record travels as under PT, or 0 when it stays a record."""
    if int(rec["kind"]) != abi.CESC_PLAN:
        return 0
    n, F = co.n, co.F
    r, rest = divmod(int(rec["slot"]), n * F)
    g, f = divmod(rest, F)
    meta = int(rec["meta"])
    kind, hb, count, inc = meta & 0xF, (meta >> 4) & 1, (meta >> 16) & 0xFFFF, meta >> 32
    if kind != abi.PLAN_AE or inc != int(co.incarnation[g]) or int(rec["e"]) != int(co.epoch[g]["x"]) or count >= 64:
        return 0
    prev, prev_term, last, commit = int(rec["a"]), int(rec["b"]), int(rec["c"]), int(rec["d"])
    gap = (int(co.current_term[g]) - prev_term) & M64
    dprev = (int(co.last_entry[g]["x"]) - prev) & M64
    dcommit = (int(co.commit_index[g]) - commit) & M64
    if not (1 <= gap <= 8) or last != ((prev + count + (1 << 63)) & M64) - (1 << 63) or dprev >= 256 or dcommit >= 16:
        return 0
    tag = (int(co.plan_c[r, g, f]) >> 5) & 63                              # the tag the plan took, as for kind 1
    return abi.CPLAN_AE_PREV_TERM | (hb << 3) | (tag << 5) | (count << 11) | (dprev << 17) | ((gap - 1) << 25) | (dcommit << 28)


def prev_term_words(co: compact.CompactOutbox, esc_cap: int) -> compact.CompactOutbox:
    """pack_kernel<.., PT = true> from pack_kernel<.., false>: co is a compact outbox packed WITHOUT the flag whose escape list
    did not overflow; every plan record that fits kind 7 becomes its word again.  The flag changes no tag: a plan takes and
    parks its tag whether it travels as a word or a record."""
    if int(co.counts[0]) > co.esc_cap:
        raise OverflowError("the unflagged escape list overflowed")
    out = compact.CompactOutbox(co.rows, co.n, co.F, esc_cap=esc_cap)
    for name in compact.CompactOutbox.COLS:
        getattr(out, name)[...] = getattr(co, name)
    out.counts[:] = co.counts
    keep = []
    for rec in co.esc[:int(co.counts[0])]:
        w = prev_term_word(co, rec)
        if w:
            out.plan_c.reshape(-1)[int(rec["slot"])] = w
        else:
            keep.append(rec)
    out.counts[0] = len(keep)
    for k, rec in enumerate(keep[:esc_cap]):
        out.esc[k] = rec
    return out


def unpack(ci: compact.CompactInbox, g_term: np.ndarray, st: InFlight, flags: int = 0) -> abi.Inbox:
    """unpack_kernel<EL> + unpack_escapes_kernel, and unpack_requests_kernel<EL> when the step has a request list (ci.reqs):
    a compact inbox -> the dense inbox the step kernel reads, entry pool included.  PT changes nothing on the way up (an ack
    to a kind-7 plan is an AE ack)."""
    el = bool(flags & EL)
    rows, n, F = ci.rows, ci.n, ci.F
    ib = abi.Inbox(rows, n, F)
    ib.flags = abi.INBOX_NO_REQUESTS
    ib.op_cd = None; ib.op_e = None
    if ci.ev_c is None:
        ib.ev_meta = ib.ev_tn = ib.ev_el = None
    else:
        for g in range(n):
            for f in range(F):
                b = int(st.bits[g, f])
                for r in range(rows):
                    w = int(ci.ev_c[r, g, f])
                    kind = w & 0xF
                    now = int(ci.row_base[r]) + (w >> 16)
                    if kind in (abi.EV_AE_ACK, abi.EV_IS_ACK):
                        tag = (w >> 8) & 0xFF
                        echo, inc = (0, 0), 0
                        if tag < CTAGS:
                            echo, inc = (int(st.el[tag, g, f]["x"]), int(st.el[tag, g, f]["y"])), int(st.inc[tag, g, f])
                            b &= ~(1 << tag)
                        ib.ev_meta[r, g, f] = (w & 0x7F) | (inc << 32)
                        ib.ev_tn[r, g, f] = (int(g_term[g]) if (w >> 7) & 1 else 0, now)
                        ib.ev_el[r, g, f] = echo
                    elif el and kind in (abi.EV_PV_REPLY, abi.EV_RV_REPLY):
                        tag = (w >> 8) & 0x1F
                        bt, inc = int(st.el[tag, g, f]["x"]), int(st.inc[tag, g, f])
                        b &= ~(1 << tag)
                        ok = ((w >> 4) & 3) == abi.OUT_OK
                        rt = ((bt - ((w >> 13) & 7) + (1 << 63)) % (1 << 64)) - (1 << 63) if ok else 0
                        ib.ev_meta[r, g, f] = (w & 0x7F) | (inc << 32)
                        ib.ev_tn[r, g, f] = (rt, now)
                        ib.ev_el[r, g, f] = (0, 0)
                    elif el and kind == abi.CEV_ESCAPED:
                        tag = (w >> 8) & 0xFF
                        if tag < CTAGS:
                            b &= ~(1 << tag)
                st.bits[g, f] = b
        for e in ci.esc:
            r, rest = divmod(int(e["slot"]), n * F); g, f = divmod(rest, F)
            ib.ev_meta[r, g, f] = e["ev_meta"]; ib.ev_tn[r, g, f] = (e["term"], e["now_ms"]); ib.ev_el[r, g, f] = (e["epoch_at_send"], e["last_at_send"])
    if ci.op_c is None:
        ib.op_meta = ib.op_nr = ib.op_ab = None
    else:
        c = ci.op_c.astype(np.uint64)
        ib.op_meta[:] = (c & U64(0xF)) | (((c >> U64(4)) & U64(0xFFF)) << U64(16))
        ib.op_nr["x"] = ci.row_base[:, None] + (c >> U64(16)).astype(np.int64)
        if ci.op_unavail is not None:
            ib.op_ab["x"] = ci.op_unavail.astype(np.int64)
        else:
            ib.op_ab = None
    q = getattr(ci, "reqs", None)
    if q is None:
        return ib
    ib.flags = 0
    if ib.op_meta is None:
        ib.op_meta = np.zeros((rows, n), np.uint64)
        ib.op_nr = np.zeros((rows, n), abi.I64X2)
        ib.op_nr["x"] = ci.row_base[:, None]
    if ib.op_ab is None:
        ib.op_ab = np.zeros((rows, n), abi.I64X2)
    ib.op_cd = np.zeros((rows, n), abi.I64X2)
    ib.op_e = np.zeros((rows, n), np.int64)
    counts = ((q.req["meta"] >> np.uint32(5)) & np.uint32(0x3F)).astype(np.int64)
    pool_end = len(q.ent_terms) + q.req_entries
    ib.ent_terms = np.zeros(max(pool_end, 1), np.int64)
    ib.ent_terms[:len(q.ent_terms)] = q.ent_terms
    ib.ent_count = pool_end
    offs = len(q.ent_terms) + np.concatenate([[0], np.cumsum(counts)[:-1]]).astype(np.int64) if len(q.req) else []
    rs, es = q.req["slot"].astype(np.int64), q.op_esc["slot"].astype(np.int64)
    unordered = bool((np.diff(rs) < 0).any() or (np.diff(es) < 0).any())
    op_c = ci.op_c.reshape(-1) if ci.op_c is not None else np.zeros(rows * n, np.uint32)
    claims = {}
    for s in list(rs) + list(es):
        claims[s] = claims.get(s, 0) + 1
    flat = lambda a: a.reshape(-1)

    def put(s, meta, now, draw, a, b, c, d, e):
        flat(ib.op_meta)[s] = meta
        flat(ib.op_nr)[s] = (now, draw); flat(ib.op_ab)[s] = (a, b); flat(ib.op_cd)[s] = (c, d); flat(ib.op_e)[s] = e

    wrap = lambda x: ((int(x) + (1 << 63)) % (1 << 64)) - (1 << 63)
    for j, x in enumerate(q.req):
        s = int(x["slot"])
        if s >= rows * n:
            continue
        m = int(x["meta"])
        vk = (m >> 11) & 3 if el else 0                                   # EL: meta bits 11..12 name a PreVote / RequestVote
        bad = (unordered or claims[s] > 1 or (int(op_c[s]) & 0xF) != 0 or (m & (0xE000 if el else 0xF800)) != 0 or vk == 3 or
               (vk != 0 and (int(counts[j]) != 0 or int(x["d_commit"]) != 0)))
        if bad:
            put(s, abi.COP_MALFORMED, int(ci.row_base[s // n]), 0, 0, 0, 0, 0, 0)
            continue
        term, prev = int(x["term"]), int(x["prev_index"])
        now = int(ci.row_base[s // n]) + (m >> 16)
        if vk:
            put(s, abi.op_make(abi.OP_PREVOTE_REQ if vk == abi.CREQ_VOTE_PRE else abi.OP_VOTE_REQ, m & 0x1F, 0), now, 0,
                term, prev, wrap(term - int(x["d_prev_term"])), 0, 0)
            continue
        cnt, off = int(counts[j]), int(offs[j])
        if off + cnt <= pool_end:
            ib.ent_terms[off:off + cnt] = x["term"]
        put(s, abi.op_make(abi.OP_AE_REQUEST, m & 0x1F, cnt) | (min(off, 0xFFFFFFFF) << 32), now, 0,
            term, prev, wrap(term - int(x["d_prev_term"])), wrap(prev + int(x["d_commit"])), wrap(prev + 1))
    for x in q.op_esc:
        s = int(x["slot"])
        if s >= rows * n:
            continue
        if unordered or claims[s] > 1 or (int(op_c[s]) & 0xF) != 0:
            put(s, abi.COP_MALFORMED, int(ci.row_base[s // n]), 0, 0, 0, 0, 0, 0)
            continue
        put(s, (int(x["op_meta"]) & 0xFFFFFFFF) | (int(x["ent"]) << 32), x["now_ms"], x["draw"], x["a"], x["b"], x["c"], x["d"], x["e"])
    return ib


# ---- the host side of a compact pump ----

def oracle_epoch(o, G: int) -> np.ndarray:
    """The (epoch_index, epoch_term) column of the oracle's groups: what the engine's pack reads from its group table."""
    ep = np.zeros(G, dtype=abi.I64X2)
    for g in range(G):
        s = o.export(g)
        ep[g] = (s.epoch_index, s.epoch_term)
    return ep


def assert_step_reads_the_same(a: abi.Inbox, b: abi.Inbox, where=""):
    """Every inbox column the step reads: lane events where present, and per group op what its kind uses (SUBMIT / TIMEOUT:
    time, draw and unavailable mask; requests: every field, entry terms by value)."""
    ek = (a.ev_meta & U64(0xF)) != 0
    assert np.array_equal(a.ev_meta, b.ev_meta), where
    for name in ("ev_tn", "ev_el"):
        assert np.array_equal(getattr(a, name)[ek], getattr(b, name)[ek]), f"{name} {where}"
    lo = lambda m: m & U64(0xFFFFFFFF)
    assert np.array_equal(lo(a.op_meta), lo(b.op_meta)), f"op kind / peer / count {where}"
    kind = (a.op_meta & U64(0xFF)).astype(np.int64)
    has = kind != 0
    assert np.array_equal(a.op_nr[has], b.op_nr[has]), f"op_nr {where}"
    simple = (kind == abi.OP_SUBMIT) | (kind == abi.OP_TIMEOUT)
    ua = a.op_ab["x"] if a.op_ab is not None else np.zeros(kind.shape, np.int64)
    ub = b.op_ab["x"] if b.op_ab is not None else np.zeros(kind.shape, np.int64)
    assert np.array_equal(ua[simple], ub[simple]), f"unavailable mask {where}"
    req = has & ~simple
    if req.any():
        assert np.array_equal(a.op_ab[req], b.op_ab[req]) and np.array_equal(a.op_cd[req], b.op_cd[req]), f"op_ab / op_cd {where}"
        assert np.array_equal(a.op_e[req], b.op_e[req]), f"op_e {where}"
        for r, i in np.argwhere(kind == abi.OP_AE_REQUEST):
            cnt = int(a.op_meta[r, i] >> U64(16)) & 0xFFFF
            oa, ob = int(a.op_meta[r, i] >> U64(32)), int(b.op_meta[r, i] >> U64(32))
            assert np.array_equal(a.ent_terms[oa:oa + cnt], b.ent_terms[ob:ob + cnt]), f"entry terms at {(r, i)} {where}"
            assert ob + cnt <= b.ent_count


def next_of(dense: abi.Outbox, co: compact.CompactOutbox) -> dict:
    """What a pump keeps from a step for encoding the next one, whatever flags either step carries: the tags of the RPCs in
    flight (kind-7 plans included), the term / incarnation of its plans, and the term / incarnation / tags of the ballots
    the next vote replies answer.  Only a step begun with EL hands ballots tags; without it every ballot tag is CTAG_NONE
    and its replies travel in full."""
    return dict(tags=co.tags(rpc_only=True), sent_term=co.current_term.copy(), sent_inc=co.incarnation.copy(),
                ballot_term=dense.ballot_term.copy(), ballot_inc=dense.ballot_meta >> U64(32), ballot_tags=co.ballot_tags())


def encode(ib: abi.Inbox, nxt: dict | None, flags: int, *, empty_list: bool) -> compact.CompactInbox:
    """The compact inbox of a step begun with `flags`, from what next_of kept of the last step (None: there was none).
    empty_list: a step whose inbox holds no request still gets a request list, an empty one, so its replies may travel in
    rep_c; otherwise such a step has none (ci.reqs is None) and every reply is an escape record."""
    ci = compact.encode_inbox(ib, **(nxt or dict(tags=None, sent_term=None)), elections=bool(flags & EL))
    if empty_list and ci.reqs is None:
        ci.reqs = compact.CompactRequests()
    return ci


def _storm_open(G, R, rows):
    """Config #3: G groups at follower slot 1, at mixed terms and log ends; its cfg, group init and vote storm workload."""
    cfg = abi.make_cfg(replicas=R, local_slot=1, max_groups=G, max_rows=rows, entry_pool_cap=workload.POOL_TERMS)
    init = harness.init_array(G, terms=1 + np.arange(G) % 5)
    init["last_index"] = 100 + np.arange(G) % 50
    init["last_term"] = 1 + np.arange(G) % 5
    return cfg, init, workload.make_wl(0x5EED0003, rows, G, R - 1, local_slot=1)


def storm(G, R, rows):
    """The oracle opened at config #3, and the vote storm's workload."""
    cfg, init, w = _storm_open(G, R, rows)
    o = binding.Oracle(cfg)
    o.open_bulk(0, init)
    return o, w


class Ratios:
    """How much of a stream's election traffic travelled compact."""

    def __init__(self):
        self.replies = self.reply_words = self.ballots = self.ballot_lanes = self.vote_reqs = self.vote_records = 0
        self.ae = self.ae_records = 0

    def add(self, ib: abi.Inbox, ci: compact.CompactInbox, dense: abi.Outbox, co: compact.CompactOutbox):
        ek = (ib.ev_meta & U64(0xF)).astype(np.int64)
        self.replies += int(((ek == abi.EV_PV_REPLY) | (ek == abi.EV_RV_REPLY)).sum())
        wk = (ci.ev_c & np.uint32(0xF)).astype(np.int64)
        self.reply_words += int(((wk == abi.EV_PV_REPLY) | (wk == abi.EV_RV_REPLY)).sum())
        self.ballots += int((dense.ballot_meta != 0).sum())
        self.ballot_lanes += int(((co.plan_c[:, :, 0] & np.uint32(7)) >= abi.CPLAN_PREVOTE).sum())
        ok = (ib.op_meta & U64(0xFF)).astype(np.int64)
        self.vote_reqs += int(((ok == abi.OP_PREVOTE_REQ) | (ok == abi.OP_VOTE_REQ)).sum())
        self.ae += int((ok == abi.OP_AE_REQUEST).sum())
        if ci.reqs is not None:
            vk = (ci.reqs.req["meta"] >> np.uint32(11)) & np.uint32(3)
            self.vote_records += int((vk != 0).sum())
            self.ae_records += int((vk == 0).sum())

    def assert_mostly_compact(self, votes=True):
        if votes:
            assert self.replies > 500 and self.ballots > 100 and self.vote_reqs > 100, vars(self)
            assert self.reply_words >= 0.9 * self.replies, vars(self)
            assert self.ballot_lanes >= 0.9 * self.ballots, vars(self)
            assert self.vote_records >= 0.9 * self.vote_reqs, vars(self)


def _sorted_esc(co):
    esc = co.esc[:int(co.counts[0])].copy()
    return np.sort(esc, order=["kind", "slot"]).tobytes()


class Driver:
    """A pump around the engine (-m gpu), checked against the oracle every step, on config #3 (storm: a vote storm at
    follower slot 1) or config #5 (elected leaders, the mixed stream).  With twin, an unflagged twin engine runs the same
    stream, and prev_term_words must turn its outbox into the flagged engine's plan_c and escape records bit for bit."""

    def __init__(self, G, R, rows, storm: bool, twin: bool = False):
        from rafting_b200 import engine
        F = R - 1
        if storm:
            cfg, init, self.w = _storm_open(G, R, rows)
        else:
            cfg = abi.make_cfg(replicas=R, max_groups=G, max_rows=rows, entry_pool_cap=rows * G * 50)
            init = harness.init_array(G, terms=np.arange(G) % 7)
            self.w = workload.make_wl(0x5EED0005, rows, G, F)
        es, self.o = [engine.Engine(cfg) for _ in range(2 if twin else 1)], binding.Oracle(cfg)
        for s in es + [self.o]:
            s.open_bulk(0, init)
        if not storm:
            w1 = workload.make_wl(0x5EED0005, 1, G, F)
            want = harness.elect_all(self.o, w1)
            for e in es:
                harness.assert_outbox_equal(want, harness.elect_all(e, w1), where="election (dense path)")
        self.e, self.twin = es[0], (es[1] if twin else None)
        self.G, self.F, self.rows, self.storm = G, F, rows, storm
        self.nxt, self.prev = None, None
        self.ae = self.ae_words = self.kind7 = self.records = self.records0 = 0

    def inbox(self, k):
        """Step k of the stream, after the last step's outbox."""
        return (workload.vote_inbox_host if self.storm else workload.mixed_inbox_host)(self.w, k, self.prev)

    def step(self, ib, flags, *, empty_list: bool, esc_cap=None, where=""):
        rows, G, F = self.rows, self.G, self.F
        want = self.o.step(ib, threads=8)
        cap = rows * G * F + 2 * rows * G if esc_cap is None else esc_cap
        cin = encode(ib, self.nxt, flags, empty_list=empty_list)
        cout = compact.CompactOutbox(rows, G, F, esc_cap=cap)
        self.e.step_compact(cin, cout, reqs=cin.reqs, flags=flags)
        if self.twin is not None:
            cout0 = compact.CompactOutbox(rows, G, F, esc_cap=rows * G * F + 2 * rows * G)
            self.twin.step_compact(cin, cout0, reqs=cin.reqs, flags=flags & ~PT)
            model = prev_term_words(cout0, cap) if flags & PT else cout0
            assert np.array_equal(cout.plan_c, model.plan_c), f"plan_c differs from the model, {where}"
            assert np.array_equal(cout.tags(), model.tags()) and np.array_equal(cout.tags(rpc_only=True), model.tags(rpc_only=True))
            assert np.array_equal(cout.counts, model.counts) and _sorted_esc(cout) == _sorted_esc(model), f"escape records, {where}"
            self.records0 += int((cout0.esc[:int(cout0.counts[0])]["kind"] == abi.CESC_PLAN).sum())
        if esc_cap is None:
            harness.assert_outbox_equal(want, compact.decode_outbox(cout, elections=bool(flags & EL), prev_term=bool(flags & PT)),
                                        where=where)
            k = cout.plan_c & np.uint32(7)
            esc = ((cout.plan_c >> np.uint32(4)) & np.uint32(1)) != 0
            self.ae += int(((want.plan_meta & np.uint64(0xF)) == abi.PLAN_AE).sum())
            self.ae_words += int((((k == abi.PLAN_AE) & ~esc) | (k == abi.CPLAN_AE_PREV_TERM)).sum())
            self.kind7 += int((k == abi.CPLAN_AE_PREV_TERM).sum())
            self.records += int((cout.esc[:int(cout.counts[0])]["kind"] == abi.CESC_PLAN).sum())
        self.nxt, self.prev = next_of(want, cout), want
        return cin, want, cout
