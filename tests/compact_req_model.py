"""numpy restatement of the request-list half of the engine's compact kernels (rafting_b200/csrc/compact.cuh:
creq_prepare_kernel + unpack_requests_kernel, and pack_kernel's compact replies) — TEST INFRASTRUCTURE beside
tests/compact_model.py, whose unpack / pack it builds on: the CPU suite uses it to check that the request list of
include/rafting_b200.h is lossless without a GPU; under -m gpu the real kernels are checked against the oracle
(tests/test_compact_requests_gpu.py)."""
from __future__ import annotations

import numpy as np

from rafting_b200 import abi, compact
from tests.compact_model import InFlight, pack, unpack


def pack_req(dense: abi.Outbox, epoch: np.ndarray, st: InFlight, esc_cap: int) -> compact.CompactOutbox:
    """pack_kernel of a step begun with a request list: as pack(), and a valid reply whose term is the group's end-of-step
    term travels in rep_c (bit 7, success in bit 6) instead of the escape list."""
    rows, n = dense.rows, dense.n
    co = pack(dense, epoch, st, esc_cap=rows * n * dense.F + 2 * rows * n)       # room for every record
    esc = co.esc[:int(co.counts[0])]
    keep = np.ones(len(esc), dtype=bool)
    for k, rec in enumerate(esc):
        if int(rec["kind"]) != abi.CESC_REPLY:
            continue
        r, g = divmod(int(rec["slot"]), n)
        rm = int(rec["meta"])
        if int(rec["a"]) == int(dense.current_term[g]):
            co.rep_c[r, g] |= 0x80 | (((rm >> 1) & 1) << 6)
            keep[k] = False
    esc = esc[keep]
    out = compact.CompactOutbox(rows, n, dense.F, esc_cap=esc_cap)
    for name in compact.CompactOutbox.COLS:
        getattr(out, name)[...] = getattr(co, name)
    out.counts[:] = co.counts
    out.counts[0] = len(esc)
    out.esc[:min(len(esc), esc_cap)] = esc[:esc_cap]
    return out


def unpack_req(ci: compact.CompactInbox, g_term: np.ndarray, st: InFlight) -> abi.Inbox:
    """unpack_kernel + unpack_escapes_kernel + unpack_requests_kernel: a compact inbox with its request list (ci.reqs) ->
    the dense inbox the step kernel reads, entry pool included."""
    ib = unpack(ci, g_term, st)
    q = ci.reqs
    if q is None:
        return ib
    rows, n = ci.rows, ci.n
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
        bad = unordered or claims[s] > 1 or (int(op_c[s]) & 0xF) != 0 or (int(x["meta"]) & 0xF800) != 0
        if bad:
            put(s, abi.COP_MALFORMED, int(ci.row_base[s // n]), 0, 0, 0, 0, 0, 0)
            continue
        m, cnt, off = int(x["meta"]), int(counts[j]), int(offs[j])
        if off + cnt <= pool_end:
            ib.ent_terms[off:off + cnt] = x["term"]
        term, prev = int(x["term"]), int(x["prev_index"])
        put(s, abi.op_make(abi.OP_AE_REQUEST, m & 0x1F, cnt) | (min(off, 0xFFFFFFFF) << 32), int(ci.row_base[s // n]) + (m >> 16), 0,
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
