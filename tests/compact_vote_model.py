"""numpy restatement of the election half of the engine's compact kernels (rafting_b200/csrc/compact.cuh, the
RAFTING_COMPACT_ELECTIONS instantiations of unpack_kernel, pack_kernel and unpack_requests_kernel) — TEST INFRASTRUCTURE
beside tests/compact_model.py and tests/compact_req_model.py: the CPU suite uses it to check that ballots as plan_c lanes,
vote replies as ev_c words and vote records are lossless without a GPU; under -m gpu the real kernels are checked against the
oracle (tests/test_compact_elections_gpu.py)."""
from __future__ import annotations

import numpy as np

from rafting_b200 import abi, compact
from tests.compact_model import CTAGS, InFlight

U64 = np.uint64
M64 = (1 << 64) - 1


def ballot_lane_kind(dense: abi.Outbox, r: int, g: int) -> int:
    """The plan_c kind the ballot of (r, g) travels as (CPLAN_PREVOTE / CPLAN_VOTE), or 0 when it stays an escape record."""
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


def pack_el(dense: abi.Outbox, epoch: np.ndarray, st: InFlight, esc_cap: int, compact_replies: bool = True) -> compact.CompactOutbox:
    """pack_kernel<EL>: as compact_model.pack (+ compact_req_model.pack_req's rep_c when compact_replies), and a ballot that
    matches the end-of-step columns becomes one plan_c word per lane, each taking the lowest free tag of its lane in row
    order, interleaved with the AE / IS plans of the same lane."""
    rows, n, F = dense.rows, dense.n, dense.F
    co = compact.CompactOutbox(rows, n, F, esc_cap=esc_cap)
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
                    if bkind[r, g]:
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
                if compact_replies and int(dense.rep_term[r, g]) == term_end:
                    co.rep_c[r, g] |= 0x80 | (((rm >> 1) & 1) << 6)
                else:
                    esc.append((abi.CESC_REPLY, r * n + g, rm, int(dense.rep_term[r, g]), 0, 0, 0, 0))
            bm = int(dense.ballot_meta[r, g])
            if bm:
                co.counts[1] += 1
                if not bkind[r, g]:
                    bl = dense.ballot_last[r, g]
                    esc.append((abi.CESC_BALLOT, r * n + g, bm, int(dense.ballot_term[r, g]), int(bl["x"]), int(bl["y"]), 0, 0))
    co.counts[0] = len(esc)
    for k, rec in enumerate(esc[:esc_cap]):
        co.esc[k] = rec
    return co


def unpack_el(ci: compact.CompactInbox, g_term: np.ndarray, st: InFlight) -> abi.Inbox:
    """unpack_kernel<EL> + unpack_escapes_kernel + unpack_requests_kernel<EL>: a compact inbox (with its request list ci.reqs,
    or None) -> the dense inbox the step kernel reads."""
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
                        el, inc = (0, 0), 0
                        if tag < CTAGS:
                            el, inc = (int(st.el[tag, g, f]["x"]), int(st.el[tag, g, f]["y"])), int(st.inc[tag, g, f])
                            b &= ~(1 << tag)
                        ib.ev_meta[r, g, f] = (w & 0x7F) | (inc << 32)
                        ib.ev_tn[r, g, f] = (int(g_term[g]) if (w >> 7) & 1 else 0, now)
                        ib.ev_el[r, g, f] = el
                    elif kind in (abi.EV_PV_REPLY, abi.EV_RV_REPLY):
                        tag = (w >> 8) & 0x1F
                        bt, inc = int(st.el[tag, g, f]["x"]), int(st.inc[tag, g, f])
                        b &= ~(1 << tag)
                        ok = ((w >> 4) & 3) == abi.OUT_OK
                        rt = ((bt - ((w >> 13) & 7) + (1 << 63)) % (1 << 64)) - (1 << 63) if ok else 0
                        ib.ev_meta[r, g, f] = (w & 0x7F) | (inc << 32)
                        ib.ev_tn[r, g, f] = (rt, now)
                        ib.ev_el[r, g, f] = (0, 0)
                    elif kind == abi.CEV_ESCAPED:
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
        vk = (m >> 11) & 3
        bad = (unordered or claims[s] > 1 or (int(op_c[s]) & 0xF) != 0 or (m & 0xE000) != 0 or vk == 3 or
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
