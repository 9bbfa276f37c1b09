"""The compact kernels over an active list (rafting_step_begin_compact_active) — TEST INFRASTRUCTURE, on top of
tests/compact_model.py, which stays the one restatement of the kernels.

With an active list, one thread per (position, follower) does what the whole-shard kernel's thread does for its group: the
wire and the dense columns are positional (group columns in the RAFTING_INBOX_COMPACT_GROUPS shape), while the in-flight
table, g_term and the epoch column stay indexed by gid.  Every lane is independent of every other, so the active kernels are
the whole-shard model run over the listed gids' slice of that state:

  pack / unpack          compact_model.pack / unpack on the slice st[gids], written back afterwards
  positions / carry      what a pump kept from a step over one list, mapped by gid onto the next step's list
  carry_outbox           the same for the previous outbox the workload generators read"""
from __future__ import annotations

import numpy as np

from rafting_b200 import abi, compact
from tests import compact_model as model


def _slice(st: model.InFlight, gids) -> model.InFlight:
    g = np.asarray(gids, np.int64)
    s = model.InFlight.__new__(model.InFlight)
    s.el, s.inc, s.bits = st.el[:, g].copy(), st.inc[:, g].copy(), st.bits[g].copy()
    return s


def _write_back(st: model.InFlight, gids, s: model.InFlight):
    g = np.asarray(gids, np.int64)
    st.el[:, g], st.inc[:, g], st.bits[g] = s.el, s.inc, s.bits


def pack(dense: abi.Outbox, epoch: np.ndarray, st: model.InFlight, esc_cap: int, flags: int = 0, replies: bool = False,
         gids=None) -> compact.CompactOutbox:
    """pack_kernel<EL, PT, AL>: dense is positional (COMPACT_GROUPS group columns); epoch and st are by gid.  gids=None is
    compact_model.pack itself."""
    if gids is None:
        return model.pack(dense, epoch, st, esc_cap, flags=flags, replies=replies)
    s = _slice(st, gids)
    co = model.pack(dense, epoch[np.asarray(gids, np.int64)], s, esc_cap, flags=flags, replies=replies)
    _write_back(st, gids, s)
    co.gids = np.ascontiguousarray(gids, dtype=np.uint32)
    return co


def unpack(ci: compact.CompactInbox, g_term: np.ndarray, st: model.InFlight, flags: int = 0, gids=None) -> abi.Inbox:
    """unpack_kernel<EL, AL> + the positional request and escape kernels: g_term and st are by gid; the dense inbox carries
    the list with RAFTING_INBOX_COMPACT_GROUPS, as the engine sets it.  gids=None is compact_model.unpack itself."""
    if gids is None:
        return model.unpack(ci, g_term, st, flags=flags)
    s = _slice(st, gids)
    ib = model.unpack(ci, g_term[np.asarray(gids, np.int64)], s, flags=flags)
    _write_back(st, gids, s)
    ib.gids = np.ascontiguousarray(gids, dtype=np.uint32)
    ib.flags |= abi.INBOX_COMPACT_GROUPS
    return ib


def positions(frm, to, G: int) -> np.ndarray:
    """For each position of the list `to`, the position its gid holds in the list `frm` (-1: not there); None = whole shard."""
    f = np.arange(G) if frm is None else np.asarray(frm, np.int64)
    t = np.arange(G) if to is None else np.asarray(to, np.int64)
    at = np.full(G, -1, np.int64)
    at[f] = np.arange(len(f))
    return at[t]


def carry(nxt: dict, frm, to, G: int) -> dict:
    """What compact_model.next_of kept from a step over the list frm, for a step over the list to: every per-position array
    follows its gid.  A gid the last step did not hold has no RPC and no ballot in flight from it (CTAG_NONE, zeros)."""
    p = positions(frm, to, G)
    has, q = p >= 0, np.maximum(p, 0)
    out = {}
    for k, v in nxt.items():
        axis = 0 if v.ndim == 1 else 1
        x = np.take(v, q, axis=axis)
        idx = (~has,) if axis == 0 else (slice(None), ~has)
        x[idx] = abi.CTAG_NONE if k in ("tags", "ballot_tags") else 0
        out[k] = x
    return out


def carry_outbox(o: abi.Outbox, frm, to, G: int) -> abi.Outbox:
    """The outbox of a step over the list frm (group columns by position, or [G] by gid for the whole shard) as the previous
    outbox of a step over the list to, for the workload generators: rows and group columns follow their gid, zeros where the
    gid was not in frm."""
    p = positions(frm, to, G)
    has, q = p >= 0, np.maximum(p, 0)
    n = G if to is None else len(to)
    out = abi.Outbox(o.rows, n, o.F, n)
    for name, _, _ in abi.Outbox.ROW_COLS:
        x = np.take(getattr(o, name), q, axis=1)
        x[:, ~has] = 0
        getattr(out, name)[...] = x
    for name, _ in abi.Outbox.GROUP_COLS:
        x = np.take(getattr(o, name), q, axis=0)
        x[~has] = 0
        getattr(out, name)[...] = x
    return out
