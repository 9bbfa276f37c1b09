"""Synthetic replication streams (ctypes over rafting_wl_* in librafting_workload.so — a library of its own: the
simulated peers are test / bench infrastructure, not part of the product library).

Concretises BASELINE.json's one-line configs; see rafting_b200/csrc/workload.cu.  The host entry
points run on the CPU (no CUDA call is made), the device ones launch a generator kernel so the
stream is produced directly in HBM.
"""
from __future__ import annotations

import ctypes as C

from . import _build, abi

_WL = None

T0_MS = 1_700_000_000_000


class WlCfg(C.Structure):
    _fields_ = [
        ("seed", C.c_uint64), ("rows", C.c_uint32), ("n", C.c_uint32), ("F", C.c_uint32), ("gid_base", C.c_uint32),
        ("max_submit", C.c_uint32), ("p_reject_ppm", C.c_uint32), ("p_error_ppm", C.c_uint32),
        ("p_cancel_ppm", C.c_uint32), ("t0", C.c_int64), ("local_slot", C.c_uint32), ("_pad", C.c_uint32),
    ]


def make_wl(seed, rows, n, F, gid_base=0, max_submit=4, p_reject_ppm=20_000, p_error_ppm=5_000,
            p_cancel_ppm=5_000, t0=T0_MS, local_slot=0) -> WlCfg:
    """Defaults = config #2 of SURVEY.md §8(d): 97 % ok/success, 2 % ok/reject, 0.5 % error, 0.5 % canceled."""
    w = WlCfg()
    w.seed, w.rows, w.n, w.F, w.gid_base = seed, rows, n, F, gid_base
    w.max_submit, w.p_reject_ppm, w.p_error_ppm, w.p_cancel_ppm, w.t0 = max_submit, p_reject_ppm, p_error_ppm, p_cancel_ppm, t0
    w.local_slot = local_slot
    return w


def _bind():
    global _WL
    if _WL is None:
        _WL = C.CDLL(_build.build_workload())
    L = _WL
    if not getattr(L, "_wl_bound", False):
        L.rafting_wl_leader_step.argtypes = [C.POINTER(WlCfg), C.c_uint64, C.POINTER(abi.OutboxC), C.POINTER(abi.InboxC),
                                             C.c_int, C.c_void_p]
        L.rafting_wl_election_step.argtypes = [C.POINTER(WlCfg), C.c_uint32, C.POINTER(abi.OutboxC), C.POINTER(abi.InboxC),
                                               C.c_int, C.c_void_p]
        for fn in (L.rafting_wl_vote_step, L.rafting_wl_mixed_step):
            fn.argtypes = [C.POINTER(WlCfg), C.c_uint64, C.POINTER(abi.OutboxC), C.POINTER(abi.InboxC), C.c_int, C.c_void_p]
        L.rafting_wl_fill_term_pool.argtypes = [C.c_void_p, C.c_uint32, C.c_int, C.c_void_p]
        L._wl_bound = True
    return L


def leader_step(w: WlCfg, step: int, prev_out_c, inbox_c, on_device=False, stream=0):
    rc = _bind().rafting_wl_leader_step(C.byref(w), step, None if prev_out_c is None else C.byref(prev_out_c),
                                        C.byref(inbox_c), 1 if on_device else 0, C.c_void_p(stream))
    if rc:
        raise RuntimeError(f"rafting_wl_leader_step rc={rc}")


def election_step(w: WlCfg, phase: int, prev_out_c, inbox_c, on_device=False, stream=0):
    rc = _bind().rafting_wl_election_step(C.byref(w), phase, None if prev_out_c is None else C.byref(prev_out_c),
                                          C.byref(inbox_c), 1 if on_device else 0, C.c_void_p(stream))
    if rc:
        raise RuntimeError(f"rafting_wl_election_step rc={rc}")


def _over(w: WlCfg, gids) -> tuple[WlCfg, dict]:
    """w over the active list gids (None: w itself): a copy with n = len(gids), and the Inbox arguments of such a step.  The
    inbox carries RAFTING_INBOX_COMPACT_GROUPS, so the previous outbox's group columns are read by position, as a compact
    active step returns them; every draw stays keyed by the gid, so a group sees the same stream with or without a list."""
    if gids is None:
        return w, {}
    v = WlCfg()
    C.pointer(v)[0] = w
    v.n = len(gids)
    return v, dict(gids=gids)


def _listed(ib: abi.Inbox) -> abi.Inbox:
    if ib.gids is not None:
        ib.flags |= abi.INBOX_COMPACT_GROUPS
    return ib


def leader_inbox_host(w: WlCfg, step: int, prev_out: abi.Outbox | None, gids=None) -> abi.Inbox:
    """Host (numpy) inbox of one leader-steady-state step (over the active list gids when given, see _over)."""
    w, kw = _over(w, gids)
    ib = abi.Inbox(w.rows, w.n, w.F, **kw)
    ib.flags = abi.INBOX_NO_REQUESTS
    _listed(ib)
    ic = ib.as_c()
    ic.op_cd = None
    ic.op_e = None
    leader_step(w, step, None if prev_out is None else prev_out.as_c(), ic)
    ib.op_cd = None
    ib.op_e = None
    return ib


def election_inbox_host(w: WlCfg, phase: int, prev_out: abi.Outbox | None) -> abi.Inbox:
    ib = abi.Inbox(1, w.n, w.F)
    ib.flags = abi.INBOX_NO_REQUESTS
    ic = ib.as_c()
    election_step(w, phase, None if prev_out is None else prev_out.as_c(), ic)
    ib.op_cd = None
    ib.op_e = None
    return ib


POOL_TERMS = 256 * 50


def vote_inbox_host(w: WlCfg, step: int, prev_out: abi.Outbox | None, gids=None) -> abi.Inbox:
    """config #3 (RequestVote storm, PreVote on): one host inbox (over the active list gids when given, see _over)."""
    w, kw = _over(w, gids)
    ib = _listed(abi.Inbox(w.rows, w.n, w.F, **kw))
    rc = _bind().rafting_wl_vote_step(C.byref(w), step, None if prev_out is None else C.byref(prev_out.as_c()),
                                      C.byref(ib.as_c()), 0, None)
    if rc:
        raise RuntimeError(f"rafting_wl_vote_step rc={rc}")
    return ib


def mixed_inbox_host(w: WlCfg, step: int, prev_out: abi.Outbox | None, gids=None) -> abi.Inbox:
    """config #5 (mixed leader churn + InstallSnapshot catch-up): one host inbox (over the active list gids when given, see
    _over)."""
    w, kw = _over(w, gids)
    ib = _listed(abi.Inbox(w.rows, w.n, w.F, ent_cap=POOL_TERMS, **kw))
    _bind().rafting_wl_fill_term_pool(ib.ent_terms.ctypes.data, POOL_TERMS, 0, None)
    ib.ent_count = POOL_TERMS
    rc = _bind().rafting_wl_mixed_step(C.byref(w), step, None if prev_out is None else C.byref(prev_out.as_c()),
                                       C.byref(ib.as_c()), 0, None)
    if rc:
        raise RuntimeError(f"rafting_wl_mixed_step rc={rc}")
    return ib
