"""numpy restatement of the engine's compact kernels (rafting_b200/csrc/compact.cuh) and the host side of a compact pump
around it — TEST INFRASTRUCTURE.

  pack / unpack      pack_kernel<EL, PT>, and unpack_kernel<EL> + unpack_escapes_kernel + unpack_requests_kernel<EL>, keyed by
                     the step's flags word (abi.COMPACT_ELECTIONS = EL, abi.COMPACT_PREV_TERM = PT) as the kernels are
  prev_term_words    the only restatement of the kind-7 rule: what PT changes in a packed outbox
  encode / next_of   what a pump encodes a step's inbox with, and what it keeps from the step for the next one
  Driver             such a pump around the engine, checked against the oracle every step (-m gpu)
  FuzzPump           harness.Fuzzer's streams through the codec and the model, and the engine with -m gpu, on the matrix
                     COMPACT_FUZZ (tests/test_compact_fuzz_{cpu,gpu}.py)

The CPU suites (tests/test_compact_*_cpu.py) run the model around the oracle to check that the compact wire format of
include/rafting_b200.h is lossless without a GPU; under -m gpu the real kernels are checked against the oracle and the
model (tests/test_compact_*_gpu.py)."""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np
import pytest

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
    ok = ek & (((a.ev_meta >> U64(4)) & U64(3)) == abi.OUT_OK)         # a reply's term is read only when it came back OK
    assert np.array_equal(a.ev_meta, b.ev_meta), where
    assert np.array_equal(a.ev_tn["y"][ek], b.ev_tn["y"][ek]) and np.array_equal(a.ev_tn["x"][ok], b.ev_tn["x"][ok]), f"ev_tn {where}"
    assert np.array_equal(a.ev_el[ek], b.ev_el[ek]), f"ev_el {where}"
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


# ---- the fuzz pump: harness.Fuzzer's streams through the compact host path ----

@dataclass(frozen=True)
class CompactCase(harness.FuzzCase):
    """A harness.FuzzCase on the compact host path.  n_active: the host's list (tail stays 0: a compact list holds gids below
    max_groups only); for a due step the device appends up to `cap` more.
      entry      whole: rafting_step_begin_compact / _req (flags 0) or _ex; active: _active over the list; sweep: _sweep over
                 the whole shard, active-sweep: over the list; due: _due over the list, one sweep row per step
      cflags     the compact step's flags (EL, PT)
      cfg_flags  the engine's cfg.flags
      esc_step   the step that runs with an escape list of ESC_SMALL records: it overflows, and the dense fetch stands in"""
    entry: str = "whole"
    cflags: int = 0
    cfg_flags: int = 0
    esc_step: int = 2

    def cfg(self) -> abi.Cfg:
        return abi.make_cfg(replicas=self.R, local_slot=self.local_slot, max_groups=self.G, max_rows=self.rows,
                            pre_vote=self.pre_vote, entry_pool_cap=self.rows * self.G * 8, flags=self.cfg_flags)

    @property
    def listed(self) -> bool:
        return self.entry in ("active", "active-sweep", "due")


def _c(id, R, G, seed, entry, cflags=0, sorted_=False, **kw):
    sweep = {"sweep": 7, "active-sweep": 5, "due": kw.get("rows", 3)}.get(entry, 0)
    steps = dict(steps=10, cpu_steps=4, leader_share=0.35, state_every=5) if sorted_ else dict(steps=16, cpu_steps=6, state_every=5)
    steps.update(kw)
    return CompactCase(id, R, G, seed, entry=entry, cflags=cflags, sweep_every=sweep, stray=4, **steps)


ESC_SMALL = 4
CFG_BOTH = abi.CFG_STRICT_CANDIDATE_VOTE | abi.CFG_LENIENT_FOLLOWER_COMMIT

# R = 2, 3, 5, 9, 17 (every step kernel the compact path reaches), unsorted (n < 2048) and class-sorted (n >= 2048 with
# requests, steady leaders elected first), every entry point, the flags spread over the cases, wide values on about half
COMPACT_FUZZ = [
    _c("R2-G777-whole", 2, 777, 61, "whole", local_slot=1),
    _c("R2-active2100-EL-wide", 2, 4096, 62, "active", EL, sorted_=True, n_active=2100, compact=True, wide=True),
    _c("R3-G777-whole-ELPT-wide", 3, 777, 63, "whole", EL | PT, wide=True),
    _c("R3-G2304-sweep-PT", 3, 2304, 64, "sweep", PT, sorted_=True, local_slot=1),
    _c("R3-G777-due", 3, 777, 65, "due", n_active=300, compact=True, local_slot=2),
    _c("R5-G777-sweep-EL-strict-lenient", 5, 777, 66, "sweep", EL, local_slot=2, cfg_flags=CFG_BOTH),
    _c("R5-active2100-sweep-ELPT-wide", 5, 4096, 67, "active-sweep", EL | PT, sorted_=True, n_active=2100, compact=True,
       wide=True, local_slot=4),
    _c("R9-G600-due-ELPT-wide", 9, 600, 68, "due", EL | PT, n_active=200, compact=True, wide=True, local_slot=8),
    _c("R9-G2304-whole-PT", 9, 2304, 69, "whole", PT, sorted_=True, local_slot=3),
    _c("R17-G300-whole-EL-wide", 17, 300, 70, "whole", EL, wide=True),
    _c("R17-active200-sweep-PT", 17, 300, 71, "active-sweep", PT, n_active=200, compact=True, local_slot=16),
]


class StreamCoverage:
    """Where a case's stream went, through the codec: per-step launches, roles, reply error codes, event kinds as words and
    as escape records, kind-7 words, compact ballot lanes, events whose time lay beyond the 16-bit offset of their row, and
    AppendEntries records of groups whose log lies beyond 2^32 with a leader commit above the group's own (wide_records:
    the record's prev + d_commit then moves the follower's commit index).
    Not among them: a (group, follower) lane with all 32 tags in flight.  A leader keeps at most IN_FLIGHT_LIMIT = 20 RPCs
    in flight per follower (Leadership.java:11), and in these streams a lane holds at most 21 busy tags; a lane runs out
    only when leaders step down and are elected again while their old tags go unanswered (tests/test_group_edit_gpu.py
    reaches it through reopened gids)."""

    def __init__(self):
        self.launches, self.roles, self.errs = set(), set(), set()
        self.words, self.escaped = set(), set()
        self.kind7 = self.ballot_lanes = self.far = self.wide_records = self.overflows = self.due_over = self.due_under = 0


class FuzzPump:
    """harness.Fuzzer's inboxes through the compact host path, against the oracle stepping the dense inbox into a poisoned
    outbox.  Every step:
      * the dense inbox is encoded (compact.encode_inbox) and the model's unpack must read it the same
        (assert_step_reads_the_same), over the model's own in-flight table;
      * the model's pack of the oracle's outbox, decoded, must equal that outbox;
      * with an engine (-m gpu), the engine steps the compact inbox through the case's entry point, and (a) its decoded
        outbox equals the oracle's, (b) its raw outbox equals the model's pack word for word, (c) under PT an unflagged twin
        engine's outbox through prev_term_words equals it, (d) a spread of groups' state equals the oracle's every
        state_every steps, every group's at the end.
    A reply the fuzz sends may answer a plan of any earlier step and row, so the pump finds the tag each reply echoes in the
    model's in-flight table (the lowest busy tag of the lane whose parked echo pair and incarnation match; under EL a ballot
    tag of the reply's incarnation for a vote reply) instead of taking the tags of the last step by slot.  A reply that
    matches no tag, or a forged or stale one, goes in as the encoder decides."""

    def __init__(self, case: CompactCase, engine: bool = False):
        self.case, self.cfg = case, case.cfg()
        G, F = case.G, case.R - 1
        self.G, self.F, self.rows = G, F, case.rows
        self.ref = harness.OracleSUT(self.cfg)
        init = case.init()
        self.ref.open_bulk(0, init)
        self.e = self.twin = None
        if engine:
            from rafting_b200 import engine as eng
            self.e = eng.Engine(self.cfg)
            self.e.open_bulk(0, init)
            if case.cflags & PT:
                self.twin = eng.Engine(self.cfg)
                self.twin.open_bulk(0, init)
        self.st = InFlight(G, F)
        self.ballot = np.zeros((CTAGS, G, F), bool)                 # the tag parks a ballot (EL), not an AE / IS plan
        states = [self.ref.export(g) for g in range(G)]
        self.term = np.array([s.current_term for s in states], np.int64)
        self.inc = np.array([s.incarnation for s in states], np.uint32)
        self.commit = np.array([s.commit_index for s in states], np.int64)
        self.out = None
        if case.leader_share:
            w1 = workload.make_wl(case.seed, 1, G, F, local_slot=case.local_slot)
            self.out = harness.elect_all(self.ref, w1)
            for e in (self.e, self.twin):
                if e is not None:
                    harness.assert_outbox_equal(self.out, harness.elect_all(e, w1), where=f"{case.id}: election (dense path)")
            self.term, self.inc = self.out.current_term.copy(), self.out.incarnation.copy()
            self.commit = self.out.commit_index.copy()
        self.gids = case.gids()
        self.fz = harness.Fuzzer(self.cfg, self.ref, seed=case.seed, rows=case.rows, gids=self.gids,
                                 leader_share=case.leader_share, sweep_every=case.sweep_every, stray_requests=case.stray,
                                 t0=harness.T33 if case.wide else 0, jump=40_000 if case.wide else 0, unavail_lanes=F,
                                 near_commit=case.wide)
        self.spread = np.arange(0, G, max(1, G // 97))
        self.cov = StreamCoverage()
        self.k = 0

    # -- what the pump keeps between steps: the model's in-flight table, and every group's term and incarnation --
    def answer_tags(self, ib: abi.Inbox, L: np.ndarray) -> tuple[np.ndarray, np.ndarray, np.ndarray, np.ndarray]:
        """-> (ack tags, ballot tags, ballot terms, ballot incarnations), [rows, n, F] over the step's positions L"""
        rows, n, F = ib.rows, ib.n, self.F
        tags = np.full((rows, n, F), abi.CTAG_NONE, np.uint8)
        btags = np.full((rows, n, F), abi.CTAG_NONE, np.uint8)
        bterm, binc = np.zeros((rows, n, F), np.int64), np.zeros((rows, n, F), np.uint64)
        ek = (ib.ev_meta & U64(0xF)).astype(np.int64)
        taken = {}
        el = bool(self.case.cflags & EL)
        for r, i, f in np.argwhere(ek != 0):                        # row-major: a lane's events in row order
            g, kind = int(L[i]), int(ek[r, i, f])
            vote = kind in (abi.EV_PV_REPLY, abi.EV_RV_REPLY)
            if vote and not el:
                continue
            busy = int(self.st.bits[g, f]) & ~taken.get((g, f), 0)
            inc = int(ib.ev_meta[r, i, f] >> U64(32))
            for t in range(CTAGS):
                if not (busy >> t) & 1 or int(self.st.inc[t, g, f]) != inc or bool(self.ballot[t, g, f]) != vote:
                    continue
                if vote:
                    btags[r, i, f], bterm[r, i, f], binc[r, i, f] = t, int(self.st.el[t, g, f]["x"]), inc
                elif (int(self.st.el[t, g, f]["x"]), int(self.st.el[t, g, f]["y"])) == (int(ib.ev_el[r, i, f]["x"]), int(ib.ev_el[r, i, f]["y"])):
                    tags[r, i, f] = t
                else:
                    continue
                taken[(g, f)] = taken.get((g, f), 0) | (1 << t)
                break
        return tags, btags, bterm, binc

    def _pack(self, want: abi.Outbox, L, cap: int, replies: bool) -> compact.CompactOutbox:
        from tests import compact_active_model as active
        return active.pack(want, oracle_epoch(self.ref.o, self.G), self.st, cap, flags=self.case.cflags, replies=replies, gids=L)

    def step(self):
        from tests import compact_active_model as active
        from tests import due_model as dm
        from tests import launch_model
        from tests import timers_model as tm
        case, G, F, rows, k, cov = self.case, self.G, self.F, self.rows, self.k, self.cov
        flags, where = case.cflags, f"{case.id}: step {k}"
        ib = self.fz.make(self.out)
        if case.listed:
            ib.flags |= abi.INBOX_COMPACT_GROUPS
        sweep = case.entry in ("sweep", "active-sweep", "due")
        cap = 0
        if case.entry == "due":
            until = int(ib.row_now.max())
            t = tm.table([self.ref.export(g) for g in range(G)])
            n_due = len(np.setdiff1d(np.flatnonzero(tm.due(t, until)), self.gids))
            cap = min(max(1, n_due // 2) if k % 2 else n_due + 3, G - len(self.gids))
            tail, self.n_due = dm.tail(t, self.gids, cap, until)
            cov.due_over += self.n_due > cap; cov.due_under += self.n_due <= cap
            ib = compact.due_inbox(ib, cap)
            L = np.concatenate([self.gids, tail]).astype(np.uint32)
        else:
            L = self.gids if case.listed else None
        pos = np.arange(G) if L is None else L.astype(np.int64)
        n = ib.n
        # the reference: the oracle steps the dense inbox (a due step over gids u tail, positional)
        ri = ib
        if case.entry == "due":
            ri = abi.Inbox.__new__(abi.Inbox); ri.__dict__.update(ib.__dict__); ri.gids = L
        want = self.ref.step(ri)
        # encode; the model's unpack reads what the step reads
        tags, btags, bterm, binc = self.answer_tags(ib, pos)
        ci = compact.encode_inbox(ib, tags, self.term[pos], self.inc[pos], elections=bool(flags & EL), ballot_term=bterm,
                                  ballot_inc=binc, ballot_tags=btags, sweep=sweep)
        if k % 2 == 0 and ci.reqs is None:
            ci.reqs = compact.CompactRequests()                       # an empty list: replies may travel in rep_c
        seen = compact.stands_for(ib, sweep)
        assert_step_reads_the_same(seen, active.unpack(ci, self.term, self.st, flags, gids=L), where=f"encode -> unpack, {where}")
        big = rows * n * F + 2 * rows * n
        cap_out = ESC_SMALL if k == case.esc_step else big
        mco = self._pack(want, L, cap_out, replies=ci.reqs is not None)
        if int(mco.counts[0]) > cap_out:
            cov.overflows += 1
            with pytest.raises(OverflowError):
                compact.decode_outbox(mco, elections=bool(flags & EL), prev_term=bool(flags & PT))
        else:
            harness.assert_outbox_equal(want, compact.decode_outbox(mco, elections=bool(flags & EL), prev_term=bool(flags & PT)),
                                        where=f"pack -> decode, {where}")
        if self.e is not None:
            self._engine_step(ib, ci, cap, L, want, mco, cap_out, where)
        # coverage
        has_reqs = ci.reqs is not None and (len(ci.reqs.req) or len(ci.reqs.op_esc))
        cov.launches.add(launch_model.kernels(case.R, n, 0 if has_reqs else abi.INBOX_NO_REQUESTS))
        grp = np.arange(n) if case.listed else pos
        cov.roles |= set((want.role_word[grp] & 3).tolist())
        cov.errs |= set(((want.rep_meta >> np.uint32(8)) & np.uint32(0xFF)).ravel().tolist())
        cov.words |= set((ci.ev_c & np.uint32(0xF)).ravel().tolist()) - {0, abi.CEV_ESCAPED}
        cov.escaped |= set((ci.esc["ev_meta"] & U64(0xF)).astype(np.int64).tolist())
        kinds = mco.plan_c & np.uint32(7)
        cov.kind7 += int((kinds == abi.CPLAN_AE_PREV_TERM).sum())
        cov.ballot_lanes += int(((kinds == abi.CPLAN_PREVOTE) | (kinds == abi.CPLAN_VOTE)).sum())
        ek = (ib.ev_meta & U64(0xF)) != 0
        cov.far += int((ek & (ib.ev_tn["y"] - ci.row_base[:, None, None] > 0xFFFF)).sum())
        if ci.reqs is not None and len(ci.reqs.req):
            q = ci.reqs.req[((ci.reqs.req["meta"] >> np.uint32(11)) & np.uint32(3)) == 0]
            prev = q["prev_index"].astype(np.int64)
            lc = prev + q["d_commit"].astype(np.int64)
            cov.wide_records += int(((prev >= 1 << 32) & (lc > self.commit[pos[q["slot"].astype(np.int64) % n]])).sum())
        # what the pump keeps
        kk, tg = mco.plan_c & np.uint32(7), mco.tags()
        for r in range(rows):
            at = np.argwhere(tg[r] < CTAGS)
            self.ballot[tg[r][at[:, 0], at[:, 1]], pos[at[:, 0]], at[:, 1]] = kk[r][at[:, 0], at[:, 1]] >= abi.CPLAN_PREVOTE
        self.term[pos] = want.current_term[:n] if case.listed else want.current_term
        self.inc[pos] = want.incarnation[:n] if case.listed else want.incarnation
        self.commit[pos] = want.commit_index[:n] if case.listed else want.commit_index
        self.out = want
        if self.e is not None and k % case.state_every == case.state_every - 1:
            for e in (self.e, self.twin):
                if e is not None:
                    harness.assert_states_equal(self.ref, e, self.spread.tolist(), F, where=where)
        self.k += 1
        return want

    def _engine_step(self, ib, ci, cap, L, want, mco, cap_out, where):
        F, rows, n, flags = self.F, self.rows, ib.n, self.case.cflags
        el, pt = bool(flags & EL), bool(flags & PT)

        def run(e, fl, esc_cap):
            cout = compact.CompactOutbox(rows, n, F, esc_cap=esc_cap, gids=None if L is None or self.case.entry == "due" else L)
            if self.case.entry == "due":
                e.step_compact_due(ci, cout, cap, reqs=ci.reqs, flags=fl)
                assert np.array_equal(cout.gids, L), f"the due step's tail differs from the model's, {where}"
                assert int(cout.counts[3]) == self.n_due, f"counts[3] = {int(cout.counts[3])}, {self.n_due} due, {where}"
            else:
                e.step_compact(ci, cout, reqs=ci.reqs, flags=fl)
            return cout

        cout = run(self.e, flags, cap_out)
        if int(cout.counts[0]) > cap_out:
            with pytest.raises(OverflowError):
                compact.decode_outbox(cout, elections=el, prev_term=pt)
            dense = abi.Outbox(rows, n, F, n if L is not None else self.G)
            self.e.step_fetch_dense(0, dense.as_c())
            harness.assert_outbox_equal(want, dense, where=f"dense fetch after an escape overflow, {where}")
        else:
            harness.assert_outbox_equal(want, compact.decode_outbox(cout, elections=el, prev_term=pt), where=f"(a) {where}")
        # (b) the raw compact outbox against the model's pack of the oracle's outbox
        assert np.array_equal(cout.plan_c, mco.plan_c), f"(b) plan_c differs from the model, {where}: {np.argwhere(cout.plan_c != mco.plan_c)[:5].tolist()}"
        assert np.array_equal(cout.rep_c, mco.rep_c), f"(b) rep_c, {where}"
        assert np.array_equal(cout.tags(), mco.tags()) and np.array_equal(cout.tags(rpc_only=True), mco.tags(rpc_only=True)), where
        assert np.array_equal(cout.counts[:3], mco.counts[:3]), f"(b) counts {cout.counts} vs {mco.counts}, {where}"
        if int(cout.counts[0]) <= cap_out:
            assert _sorted_esc(cout) == _sorted_esc(mco), f"(b) escape records, {where}"
        if self.twin is not None:                                      # (c)
            cout0 = run(self.twin, flags & ~PT, rows * n * F + 2 * rows * n)
            model = prev_term_words(cout0, cap_out)
            assert np.array_equal(cout.plan_c, model.plan_c), f"(c) plan_c, {where}"
            assert np.array_equal(cout.counts[:3], model.counts[:3]), f"(c) counts, {where}"
            if int(cout.counts[0]) <= cap_out:
                assert _sorted_esc(cout) == _sorted_esc(model), f"(c) escape records, {where}"

    def run(self, steps: int) -> StreamCoverage:
        for _ in range(steps):
            self.step()
        if self.e is not None:
            for e in (self.e, self.twin):
                if e is not None:
                    harness.assert_states_equal(self.ref, e, range(self.G), self.F, where=f"{self.case.id}: end of the run")
        return self.cov
