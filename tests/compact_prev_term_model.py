"""numpy restatement of the RAFTING_COMPACT_PREV_TERM half of the engine's pack_kernel (rafting_b200/csrc/compact.cuh, the PT
instantiations) — TEST INFRASTRUCTURE beside tests/compact_model.py, tests/compact_req_model.py and tests/compact_vote_model.py,
whose packs it builds on.  The flag changes no tag: a plan takes and parks its tag whether it travels as a word or a record.
So the flagged outbox is the unflagged one with every RAFTING_CESC_PLAN record that fits the kind-7 rule turned back into a
word (prev_term_words).  The CPU suite runs it around the oracle; under -m gpu the real kernel is checked against it."""
from __future__ import annotations

import numpy as np

from rafting_b200 import abi, compact
from tests import compact_model, compact_req_model, compact_vote_model
from tests.compact_model import InFlight

M64 = (1 << 64) - 1


def prev_term_word(co: compact.CompactOutbox, rec) -> int:
    """The kind-7 word an escaped plan record travels as under the flag, or 0 when it stays a record."""
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
    did not overflow; every plan record that fits kind 7 becomes its word again."""
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


def pack_pt(dense: abi.Outbox, epoch: np.ndarray, st: InFlight, esc_cap: int, flags: int,
            compact_replies: bool = True) -> compact.CompactOutbox:
    """pack_kernel for a step begun with `flags` (any combination of abi.COMPACT_ELECTIONS / abi.COMPACT_PREV_TERM)."""
    room = dense.rows * dense.n * dense.F + 2 * dense.rows * dense.n                 # room for every record
    if flags & abi.COMPACT_ELECTIONS:
        co = compact_vote_model.pack_el(dense, epoch, st, esc_cap=room, compact_replies=compact_replies)
    elif compact_replies:
        co = compact_req_model.pack_req(dense, epoch, st, esc_cap=room)
    else:
        co = compact_model.pack(dense, epoch, st, esc_cap=room)
    if flags & abi.COMPACT_PREV_TERM:
        return prev_term_words(co, esc_cap)
    out = compact.CompactOutbox(co.rows, co.n, co.F, esc_cap=esc_cap)
    for name in compact.CompactOutbox.COLS:
        getattr(out, name)[...] = getattr(co, name)
    out.counts[:] = co.counts
    out.esc[:min(esc_cap, int(co.counts[0]))] = co.esc[:min(esc_cap, int(co.counts[0]))]
    return out


def unpack_pt(ci: compact.CompactInbox, g_term: np.ndarray, st: InFlight, flags: int) -> abi.Inbox:
    """unpack for a step begun with `flags`: the flag changes nothing on the way up (an ack to a kind-7 plan is an AE ack)."""
    if flags & abi.COMPACT_ELECTIONS:
        return compact_vote_model.unpack_el(ci, g_term, st)
    return compact_req_model.unpack_req(ci, g_term, st)
