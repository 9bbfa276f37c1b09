"""Host-side mirror of the reference's plug points over the C ABI (librafting_b200.so).

`Engine` stands where the reference's ContextManager + the three ContextLoop threads stand
(M/context/ContextManager.java:46-106, M/support/EventLoopGroup.java:32-80): it owns every
RaftContext hosted by this node/GPU shard and drains one batch of their events per `step`.
The method names follow the reference where one exists:

    open_group / close_group   ContextManager.createContext / exitContext (+ RaftContext.initialize)
    step(inbox) -> outbox      one turn of every group's ContextEventLoop
    export(gid)                RaftContext.participant() / RaftLog.{epoch,last,lastCommitted} / Leadership.State
    log_term(gid, i)           RaftLog.get(i).term()
    allgather_commit()         (new) cross-shard commitIndex summary

This module is ctypes only: no torch, no numpy math on the data path, and NO CPU FALLBACK — if the
shared library or a CUDA device is missing it raises.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

from . import abi

_LIB = None
# RAFTING_B200_LIB selects another build of the same ABI (a copy under another name, an A/B variant)
_LIB_PATH = os.environ.get("RAFTING_B200_LIB") or os.path.join(os.path.dirname(os.path.abspath(__file__)), "librafting_b200.so")

STATUS = {0: "OK", -1: "E_INVAL", -2: "E_NOMEM", -3: "E_CUDA", -4: "E_CLOSED", -5: "E_CAPACITY",
          -6: "E_NODEVICE", -7: "E_BUSY", -8: "E_NCCL"}

EXPORTS = [
    "rafting_abi_version", "rafting_last_error", "rafting_engine_create", "rafting_engine_destroy",
    "rafting_group_open", "rafting_group_open_bulk", "rafting_group_load_runs", "rafting_group_close", "rafting_group_edit_begin", "rafting_lease", "rafting_lease_ex", "rafting_lease_release", "rafting_step",
    "rafting_step_begin", "rafting_step_wait", "rafting_step_device", "rafting_state_export",
    "rafting_state_export_bulk", "rafting_state_digest", "rafting_log_term", "rafting_commit_slice",
    "rafting_comm_init", "rafting_comm_init_all", "rafting_comm_unique_id", "rafting_allgather_commit", "rafting_allgather_commit_from",
    "rafting_allgather_commit_all", "rafting_allgather_last", "rafting_restore_async", "rafting_state_save", "rafting_state_load", "rafting_step_device_seq", "rafting_engine_stream",
    "rafting_engine_counters", "rafting_abi_sizes", "rafting_checkpoint", "rafting_restore",
    "rafting_step_begin_host", "rafting_step_wait_slot", "rafting_step_begin_compact", "rafting_step_begin_compact_req", "rafting_step_begin_compact_ex", "rafting_step_begin_compact_active", "rafting_step_begin_compact_sweep", "rafting_step_begin_compact_due", "rafting_timers_due_begin", "rafting_timers_due_wait", "rafting_compact_req_layout", "rafting_step_wait_compact", "rafting_step_fetch_dense", "rafting_compact_layout", "rafting_backoff_step", "rafting_allgather_join",
    "rafting_log_config", "rafting_log_append", "rafting_log_read", "rafting_log_gather", "rafting_log_trim", "rafting_log_stats",
    "rafting_log_gather_step_begin", "rafting_log_gather_step_wait", "rafting_log_gather_begin", "rafting_log_gather_wait",
    "rafting_log_store_open", "rafting_log_sync", "rafting_log_mark", "rafting_log_recovered", "rafting_log_export_kv", "rafting_log_store_stats",
]


class RaftingError(RuntimeError):
    def __init__(self, rc: int, what: str):
        self.rc = rc
        msg = lib().rafting_last_error().decode(errors="replace") if _LIB is not None else ""
        super().__init__(f"{what}: {STATUS.get(rc, rc)} {msg}")


def lib_path() -> str:
    return _LIB_PATH


def lib():
    """Loads the in-tree CUDA library. Raises if it has not been built (no fallback)."""
    global _LIB
    if _LIB is None:
        if not os.path.exists(_LIB_PATH):
            raise RuntimeError(
                f"{_LIB_PATH} is missing: run `python -m rafting_b200._build` (or __graft_entry__.build()). "
                "The engine has no CPU path.")
        L = C.CDLL(_LIB_PATH)
        L.rafting_abi_version.restype = C.c_uint32
        L.rafting_last_error.restype = C.c_char_p
        L.rafting_engine_create.argtypes = [C.POINTER(abi.Cfg), C.POINTER(C.c_void_p)]
        L.rafting_engine_destroy.argtypes = [C.c_void_p]
        L.rafting_group_open.argtypes = [C.c_void_p, C.c_uint32, C.POINTER(abi.GroupInit)]
        L.rafting_group_open_bulk.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p]
        L.rafting_group_close.argtypes = [C.c_void_p, C.c_uint32]
        L.rafting_group_load_runs.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32]
        L.rafting_group_edit_begin.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p]
        L.rafting_lease.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, C.POINTER(abi.LeaseC)]
        L.rafting_lease_ex.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.POINTER(abi.LeaseC)]
        L.rafting_lease_release.argtypes = [C.c_void_p, C.POINTER(abi.LeaseC)]
        L.rafting_step.argtypes = [C.c_void_p, C.POINTER(abi.LeaseC)]
        L.rafting_step_begin.argtypes = [C.c_void_p, C.POINTER(abi.LeaseC)]
        L.rafting_step_wait.argtypes = [C.c_void_p, C.POINTER(abi.LeaseC)]
        L.rafting_step_device.argtypes = [C.c_void_p, C.POINTER(abi.InboxC), C.POINTER(abi.OutboxC), C.c_void_p]
        L.rafting_state_export.argtypes = [C.c_void_p, C.c_uint32, C.POINTER(abi.GroupState)]
        L.rafting_state_export_bulk.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p]
        L.rafting_state_digest.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p]
        L.rafting_log_term.argtypes = [C.c_void_p, C.c_uint32, C.c_int64, C.POINTER(C.c_int64)]
        L.rafting_commit_slice.argtypes = [C.c_void_p, C.POINTER(C.c_void_p), C.POINTER(C.c_uint32)]
        L.rafting_comm_init.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_size_t]
        L.rafting_comm_unique_id.argtypes = [C.c_void_p, C.POINTER(C.c_size_t)]
        L.rafting_allgather_commit.argtypes = [C.c_void_p, C.c_void_p, C.POINTER(C.c_void_p)]
        L.rafting_allgather_join.argtypes = [C.c_void_p]
        L.rafting_comm_init_all.argtypes = [C.POINTER(C.c_void_p), C.c_int]
        L.rafting_allgather_commit_from.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(C.c_void_p)]
        L.rafting_allgather_commit_all.argtypes = [C.POINTER(C.c_void_p), C.c_int, C.POINTER(C.c_void_p), C.POINTER(C.c_void_p),
                                                   C.POINTER(C.c_void_p)]
        L.rafting_step_device_seq.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_int, C.c_void_p]
        L.rafting_log_config.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32]
        L.rafting_log_append.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_size_t]
        L.rafting_log_read.argtypes = [C.c_void_p, C.c_uint32, C.c_int64, C.c_uint32, C.c_void_p, C.c_void_p, C.c_size_t,
                                       C.POINTER(C.c_uint32)]
        L.rafting_log_gather.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32,
                                         C.c_void_p, C.c_size_t, C.POINTER(C.c_uint32), C.POINTER(C.c_size_t)]
        L.rafting_log_stats.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32]
        L.rafting_log_gather_step_begin.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_void_p, C.c_size_t,
                                                    C.c_void_p, C.c_uint32]
        L.rafting_log_gather_step_wait.argtypes = [C.c_void_p, C.c_uint32, C.POINTER(C.c_uint32), C.POINTER(C.c_size_t),
                                                   C.POINTER(C.c_uint32), C.POINTER(C.c_uint32)]
        L.rafting_log_gather_begin.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                               C.c_uint32, C.c_void_p, C.c_size_t]
        L.rafting_log_gather_wait.argtypes = [C.c_void_p, C.c_uint32, C.POINTER(C.c_uint32), C.POINTER(C.c_size_t),
                                              C.POINTER(C.c_uint32)]
        L.rafting_log_trim.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]
        L.rafting_log_store_open.argtypes = [C.c_void_p, C.c_char_p, C.c_uint32, C.POINTER(C.c_uint64)]
        L.rafting_log_sync.argtypes = [C.c_void_p]
        L.rafting_log_mark.argtypes = [C.c_void_p, C.c_uint32, C.c_int64, C.c_int64, C.c_int64, C.c_int64]
        L.rafting_log_recovered.argtypes = [C.c_void_p, C.c_uint32, C.POINTER(abi.GroupInit), C.c_void_p, C.c_uint32, C.POINTER(C.c_uint32)]
        L.rafting_log_export_kv.argtypes = [C.c_void_p, C.c_uint32, C.c_int64, C.c_char_p, C.c_char_p, C.c_size_t, C.POINTER(C.c_size_t)]
        L.rafting_log_store_stats.argtypes = [C.c_void_p, C.POINTER(C.c_uint64 * 6)]
        L.rafting_engine_stream.argtypes = [C.c_void_p, C.POINTER(C.c_void_p)]
        L.rafting_engine_counters.argtypes = [C.c_void_p, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]
        L.rafting_abi_sizes.argtypes = [C.POINTER(C.c_uint32), C.c_uint32]
        L.rafting_step_begin_host.argtypes = [C.c_void_p, C.c_uint32, C.POINTER(abi.InboxC), C.POINTER(abi.OutboxC)]
        L.rafting_step_wait_slot.argtypes = [C.c_void_p, C.c_uint32]
        L.rafting_step_begin_compact.argtypes = [C.c_void_p, C.c_uint32, C.POINTER(abi.CInboxC), C.POINTER(abi.COutboxC)]
        L.rafting_step_begin_compact_req.argtypes = [C.c_void_p, C.c_uint32, C.POINTER(abi.CInboxC), C.POINTER(abi.CReqsC),
                                                     C.POINTER(abi.COutboxC)]
        L.rafting_step_begin_compact_ex.argtypes = [C.c_void_p, C.c_uint32, C.POINTER(abi.CInboxC), C.POINTER(abi.CReqsC),
                                                    C.POINTER(abi.COutboxC), C.c_uint32]
        L.rafting_step_begin_compact_active.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p, C.POINTER(abi.CInboxC),
                                                        C.POINTER(abi.CReqsC), C.POINTER(abi.COutboxC), C.c_uint32]
        L.rafting_step_begin_compact_sweep.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p, C.c_void_p, C.POINTER(abi.CInboxC),
                                                       C.POINTER(abi.CReqsC), C.POINTER(abi.COutboxC), C.c_uint32]
        L.rafting_step_begin_compact_due.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p, C.c_uint32, C.c_void_p,
                                                     C.POINTER(abi.CInboxC), C.POINTER(abi.CReqsC), C.POINTER(abi.COutboxC),
                                                     C.c_void_p, C.c_uint32]
        L.rafting_timers_due_begin.argtypes = [C.c_void_p, C.c_uint32, C.c_int64, C.c_void_p, C.c_uint32]
        L.rafting_timers_due_wait.argtypes = [C.c_void_p, C.c_uint32, C.POINTER(C.c_uint32), C.POINTER(C.c_int64)]
        L.rafting_compact_req_layout.argtypes = [C.c_uint32, C.c_uint32, C.c_uint32, C.POINTER(C.c_uint64 * 4)]
        L.rafting_step_wait_compact.argtypes = [C.c_void_p, C.c_uint32]
        L.rafting_compact_layout.argtypes = [C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.POINTER(C.c_uint64 * 6),
                                             C.POINTER(C.c_uint64 * 12)]
        L.rafting_step_fetch_dense.argtypes = [C.c_void_p, C.c_uint32, C.POINTER(abi.OutboxC)]
        L.rafting_checkpoint.argtypes = [C.c_void_p]
        L.rafting_restore.argtypes = [C.c_void_p]
        L.rafting_restore_async.argtypes = [C.c_void_p]
        L.rafting_state_save.argtypes = [C.c_void_p, C.c_char_p]
        L.rafting_state_load.argtypes = [C.c_void_p, C.c_char_p]
        L.rafting_allgather_last.argtypes = [C.c_void_p, C.c_void_p]
        if L.rafting_abi_version() != abi.ABI_VERSION:
            raise RuntimeError("librafting_b200.so ABI version mismatch")
        _LIB = L
    return _LIB


def _check(rc: int, what: str):
    if rc != 0:
        raise RaftingError(rc, what)


def _np_view(ptr: int, dtype, shape):
    """numpy view over pinned host memory owned by the engine."""
    n = int(np.prod(shape)) if len(shape) else 1
    if n == 0 or not ptr:
        return np.zeros(shape, dtype=dtype)
    dt = np.dtype(dtype)
    buf = (C.c_char * (n * dt.itemsize)).from_address(ptr)
    return np.frombuffer(buf, dtype=dt, count=n).reshape(shape)


# rafting_group_init_t of a fresh, empty group: what open_group and edit_open fill in for the keywords they are not given
_INIT_DEFAULTS = dict(term=0, ballot=-1, epoch_index=0, epoch_term=0, first_index=1, last_index=0, last_term=0,
                      commit_index=0, now_ms=0, rand_ms=1000)


def edit_open(gid: int, runs=None, **kw) -> np.ndarray:
    """One OPEN record for Engine.group_edit_begin: the keywords of open_group, plus runs = [(first index, term), ...]
    oldest first as load_runs takes them (None: the single run the init describes)."""
    r = np.zeros((), dtype=abi.GROUP_EDIT)
    r["gid"], r["kind"] = gid, abi.EDIT_OPEN
    d = dict(_INIT_DEFAULTS)
    d.update(kw)
    for k, v in d.items():
        r["init"][k] = v
    if runs is not None:
        a = np.array(runs, dtype=np.int64).reshape(-1, 2)
        if len(a) > abi.TERM_RUNS:
            raise ValueError(f"{len(a)} term runs: a record holds at most {abi.TERM_RUNS}")
        r["n_runs"] = len(a)
        r["runs"][:len(a)] = np.rec.fromarrays(a.T, dtype=abi.I64X2)
    return r


def edit_close(gid: int) -> np.ndarray:
    """One CLOSE record for Engine.group_edit_begin."""
    r = np.zeros((), dtype=abi.GROUP_EDIT)
    r["gid"], r["kind"] = gid, abi.EDIT_CLOSE
    return r


class Engine:
    def __init__(self, cfg: abi.Cfg):
        self.cfg = cfg
        self.F = cfg.replicas - 1
        self.G = cfg.max_groups
        h = C.c_void_p()
        _check(lib().rafting_engine_create(C.byref(cfg), C.byref(h)), "rafting_engine_create")
        self._h = h

    def close(self):
        if getattr(self, "_h", None):
            lib().rafting_engine_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ---- lifecycle -------------------------------------------------------------------------
    def open_group(self, gid: int, **kw):
        gi = abi.GroupInit()
        d = dict(_INIT_DEFAULTS)
        d.update(kw)
        for k, v in d.items():
            setattr(gi, k, v)
        _check(lib().rafting_group_open(self._h, gid, C.byref(gi)), "rafting_group_open")

    def open_bulk(self, first_gid: int, inits: np.ndarray):
        inits = np.ascontiguousarray(inits, dtype=abi.GROUP_INIT_DTYPE)
        _check(lib().rafting_group_open_bulk(self._h, first_gid, len(inits), inits.ctypes.data), "rafting_group_open_bulk")

    def load_runs(self, gid: int, runs):
        """runs: [(first index of the run, term), ...] oldest first — the stored log's index->term map after a restart."""
        a = np.array(runs, dtype=np.int64).reshape(-1, 2)
        _check(lib().rafting_group_load_runs(self._h, gid, a.ctypes.data, len(a)), "rafting_group_load_runs")

    def close_group(self, gid: int):
        _check(lib().rafting_group_close(self._h, gid), "rafting_group_close")

    def group_edit_begin(self, edits):
        """Enqueues opens, restarts and closes (abi.GROUP_EDIT records, built by edit_open / edit_close, gids increasing) on
        the step stream, behind every step begun so far, without draining it.  The caller drops its pending RPCs of the
        edited gids: their replies must not reach a later step."""
        a = np.ascontiguousarray(np.asarray(edits, dtype=abi.GROUP_EDIT).reshape(-1))
        _check(lib().rafting_group_edit_begin(self._h, len(a), a.ctypes.data), "rafting_group_edit_begin")

    # ---- host path: lease -> fill pinned columns -> step (H2D + kernel + D2H inside) ----------
    def lease(self, rows: int, n_active: int = 0, ent_count: int = 0, flags: int = 0) -> "Lease":
        lc = abi.LeaseC()
        _check(lib().rafting_lease_ex(self._h, rows, n_active, ent_count, flags, C.byref(lc)), "rafting_lease_ex")
        compact = bool(flags & abi.INBOX_COMPACT_GROUPS)
        return Lease(self, lc, rows, n_active if n_active else self.G, gcols=n_active if compact else self.G)

    def step(self, inbox: abi.Inbox, threads: int = 1) -> abi.Outbox:
        """Same call shape as oracle.binding.Oracle.step: numpy inbox in, numpy outbox out."""
        n = inbox.n
        lease = self.lease(inbox.rows, 0 if inbox.gids is None else len(inbox.gids), inbox.ent_count,
                           inbox.flags & abi.INBOX_COMPACT_GROUPS)
        lease.fill_from(inbox)
        lease.run()
        return lease.outbox_copy()

    # ---- host path with caller-owned (pinned) buffers, two slots -------------------------------
    def step_begin_host(self, slot: int, inbox_c: abi.InboxC, outbox_c: abi.OutboxC):
        _check(lib().rafting_step_begin_host(self._h, slot, C.byref(inbox_c), C.byref(outbox_c)), "rafting_step_begin_host")

    def step_wait_slot(self, slot: int):
        _check(lib().rafting_step_wait_slot(self._h, slot), "rafting_step_wait_slot")

    # ---- compact host path: an eighth of the PCIe bytes (include/rafting_b200.h, rafting_b200/compact.py) ----------------
    def step_begin_compact(self, slot: int, cin_c: abi.CInboxC, cout_c: abi.COutboxC):
        _check(lib().rafting_step_begin_compact(self._h, slot, C.byref(cin_c), C.byref(cout_c)), "rafting_step_begin_compact")

    def step_wait_compact(self, slot: int):
        _check(lib().rafting_step_wait_compact(self._h, slot), "rafting_step_wait_compact")

    def step_fetch_dense(self, slot: int, outbox_c: abi.OutboxC):
        _check(lib().rafting_step_fetch_dense(self._h, slot, C.byref(outbox_c)), "rafting_step_fetch_dense")

    @staticmethod
    def compact_layout(rows: int, G: int, F: int, n_esc_in: int, esc_cap: int):
        """-> (in_off[6], out_off[12]) byte offsets of the wire columns inside one block per direction (rafting_compact_layout)"""
        a, b = (C.c_uint64 * 6)(), (C.c_uint64 * 12)()
        _check(lib().rafting_compact_layout(rows, G, F, n_esc_in, esc_cap, C.byref(a), C.byref(b)), "rafting_compact_layout")
        return list(a), list(b)

    def step_begin_compact_req(self, slot: int, cin_c: abi.CInboxC, reqs_c: abi.CReqsC | None, cout_c: abi.COutboxC):
        _check(lib().rafting_step_begin_compact_req(self._h, slot, C.byref(cin_c), None if reqs_c is None else C.byref(reqs_c),
                                                    C.byref(cout_c)), "rafting_step_begin_compact_req")

    @staticmethod
    def compact_req_layout(n_req: int, n_op_esc: int, ent_count: int):
        """-> byte offsets of req, op_esc, ent_terms and the block size (rafting_compact_req_layout)"""
        a = (C.c_uint64 * 4)()
        _check(lib().rafting_compact_req_layout(n_req, n_op_esc, ent_count, C.byref(a)), "rafting_compact_req_layout")
        return list(a)

    def step_begin_compact_ex(self, slot: int, cin_c: abi.CInboxC, reqs_c: abi.CReqsC | None, cout_c: abi.COutboxC, flags: int):
        _check(lib().rafting_step_begin_compact_ex(self._h, slot, C.byref(cin_c), None if reqs_c is None else C.byref(reqs_c),
                                                   C.byref(cout_c), flags), "rafting_step_begin_compact_ex")

    def step_begin_compact_active(self, slot: int, gids: np.ndarray, cin_c: abi.CInboxC, reqs_c: abi.CReqsC | None,
                                  cout_c: abi.COutboxC, flags: int = 0):
        """rafting_step_begin_compact_active: a compact step over the groups gids (uint32, strictly increasing, each below
        max_groups); every column of cin_c / cout_c holds len(gids) groups per row, by position.  gids must stay alive until
        the wait."""
        if gids.dtype != np.uint32 or not gids.flags.c_contiguous:
            raise TypeError("gids must be a contiguous uint32 array")
        _check(lib().rafting_step_begin_compact_active(self._h, slot, len(gids), gids.ctypes.data if len(gids) else None,
                                                       C.byref(cin_c), None if reqs_c is None else C.byref(reqs_c),
                                                       C.byref(cout_c), flags), "rafting_step_begin_compact_active")

    def step_begin_compact_sweep(self, slot: int, sweep: np.ndarray, cin_c: abi.CInboxC, reqs_c: abi.CReqsC | None,
                                 cout_c: abi.COutboxC, flags: int = 0, gids: np.ndarray | None = None):
        """rafting_step_begin_compact_sweep: the compact step that stands for the dense step with row_now = sweep (int64 [rows],
        0 = not a sweep row), over the whole shard (gids None) or the active list gids.  sweep and gids must stay alive until
        the wait."""
        if sweep.dtype != np.int64 or not sweep.flags.c_contiguous:
            raise TypeError("sweep must be a contiguous int64 array")
        if len(sweep) < cin_c.rows:
            raise ValueError(f"sweep holds {len(sweep)} rows, the inbox {cin_c.rows}")
        if gids is not None and (gids.dtype != np.uint32 or not gids.flags.c_contiguous):
            raise TypeError("gids must be a contiguous uint32 array")
        n, g = (0, None) if gids is None else (len(gids), gids.ctypes.data if len(gids) else None)
        _check(lib().rafting_step_begin_compact_sweep(self._h, slot, n, g, sweep.ctypes.data, C.byref(cin_c),
                                                      None if reqs_c is None else C.byref(reqs_c), C.byref(cout_c), flags),
               "rafting_step_begin_compact_sweep")

    def step_begin_compact_due(self, slot: int, gids: np.ndarray, cap: int, sweep: np.ndarray, cin_c: abi.CInboxC,
                               reqs_c: abi.CReqsC | None, cout_c: abi.COutboxC, flags: int = 0):
        """rafting_step_begin_compact_due: a sweep step over gids (uint32, strictly increasing, may be empty) followed by a tail
        of cap gids the device chooses (the groups outside gids that the sweep fires, lowest first, then groups that are not
        due).  Every column of cin_c / cout_c holds len(gids) + cap groups per row, by position; counts[3] of the outbox is the
        number of due groups outside gids.  gids and sweep must stay alive until step_wait_compact_due, which returns the tail."""
        if gids.dtype != np.uint32 or not gids.flags.c_contiguous:
            raise TypeError("gids must be a contiguous uint32 array")
        if sweep.dtype != np.int64 or not sweep.flags.c_contiguous:
            raise TypeError("sweep must be a contiguous int64 array")
        if len(sweep) < cin_c.rows:
            raise ValueError(f"sweep holds {len(sweep)} rows, the inbox {cin_c.rows}")
        if cap < 1:
            raise ValueError("cap must be at least 1")
        tail = np.zeros(cap, dtype=np.uint32)
        _check(lib().rafting_step_begin_compact_due(self._h, slot, len(gids), gids.ctypes.data if len(gids) else None, cap,
                                                    sweep.ctypes.data, C.byref(cin_c), None if reqs_c is None else C.byref(reqs_c),
                                                    C.byref(cout_c), tail.ctypes.data, flags), "rafting_step_begin_compact_due")
        self._due_tail = getattr(self, "_due_tail", {})
        self._due_tail[slot] = tail

    def step_wait_compact_due(self, slot: int) -> np.ndarray:
        """rafting_step_wait_compact for a step begun with step_begin_compact_due: -> its tail (uint32 [cap])."""
        self.step_wait_compact(slot)
        return self._due_tail.pop(slot)

    def step_compact_due(self, cin, cout, cap: int, slot: int = 0, reqs=None, flags: int = 0) -> np.ndarray:
        """Synchronous due step: cin a compact.CompactInbox encoded with sweep=True over cin.gids (the host's part, which may
        be empty) padded with cap empty positions (compact.pad_for_tail), cout a CompactOutbox of len(cin.gids) + cap groups.
        On return cout.gids is the whole list, gids followed by the tail; returns the tail."""
        host = cin.gids if cin.gids is not None else np.zeros(0, np.uint32)
        self.step_begin_compact_due(slot, host, cap, cin.sweep, cin.as_c(), None if reqs is None else reqs.as_c(), cout.as_c(), flags)
        tail = self.step_wait_compact_due(slot)
        cout.gids = np.concatenate([host, tail]).astype(np.uint32)
        return tail

    def timers_due_begin(self, slot: int, until_ms: int, out: np.ndarray | int | None, cap: int | None = None):
        """rafting_timers_due_begin: enqueue the query "which groups would a sweep at until_ms fire" behind every step begun
        so far.  out: a uint32 array (or the address of pinned host memory, with cap) that receives the due gids; it must stay
        alive until timers_due_wait."""
        if out is None:
            if cap:
                raise ValueError("a cap without a buffer")
            ptr, cap = None, 0
        elif isinstance(out, int):
            if cap is None:
                raise ValueError("an address needs its cap (the number of uint32 it holds)")
            ptr = out
        else:
            if out.dtype != np.uint32 or not out.flags.c_contiguous:
                raise TypeError("out must be a contiguous uint32 array")
            if cap is not None and cap > len(out):
                raise ValueError(f"cap {cap} exceeds the buffer's {len(out)} entries")
            ptr, cap = (out.ctypes.data if len(out) else None), len(out) if cap is None else cap
        _check(lib().rafting_timers_due_begin(self._h, slot, until_ms, ptr, cap), "rafting_timers_due_begin")

    def timers_due_wait(self, slot: int) -> tuple[int, int]:
        """-> (n_due, next_deadline_ms).  n_due may exceed the buffer's cap: then only its first cap gids were written."""
        n, nxt = C.c_uint32(), C.c_int64()
        _check(lib().rafting_timers_due_wait(self._h, slot, C.byref(n), C.byref(nxt)), "rafting_timers_due_wait")
        return n.value, nxt.value

    def timers_due(self, until_ms: int, slot: int = 0) -> tuple[np.ndarray, int]:
        """Synchronous: (the gids a sweep at until_ms would fire, the next deadline after it)."""
        out = np.zeros(self.G, dtype=np.uint32)
        self.timers_due_begin(slot, until_ms, out)
        n, nxt = self.timers_due_wait(slot)
        return out[:n].copy(), nxt

    def step_compact(self, cin, cout, slot: int = 0, reqs=None, flags: int = 0):
        """Synchronous compact step: cin / cout are rafting_b200.compact.CompactInbox / CompactOutbox, reqs a
        rafting_b200.compact.CompactRequests (None: rafting_step_begin_compact).  flags (rafting_step_begin_compact_ex):
        abi.COMPACT_ELECTIONS carries ballots, vote replies and vote requests compact, abi.COMPACT_PREV_TERM AE plans whose
        prevLogTerm lies 1..8 below the group's term; the two combine.  An inbox with an active list (cin.gids) runs through
        rafting_step_begin_compact_active, and one encoded with a sweep column (compact.encode_inbox(sweep=True)) through
        rafting_step_begin_compact_sweep."""
        if getattr(cin, "sweep", None) is not None:
            self.step_begin_compact_sweep(slot, cin.sweep, cin.as_c(), None if reqs is None else reqs.as_c(), cout.as_c(), flags,
                                          gids=getattr(cin, "gids", None))
        elif getattr(cin, "gids", None) is not None:
            self.step_begin_compact_active(slot, cin.gids, cin.as_c(), None if reqs is None else reqs.as_c(), cout.as_c(), flags)
        elif flags:
            self.step_begin_compact_ex(slot, cin.as_c(), None if reqs is None else reqs.as_c(), cout.as_c(), flags)
        elif reqs is None:
            self.step_begin_compact(slot, cin.as_c(), cout.as_c())
        else:
            self.step_begin_compact_req(slot, cin.as_c(), reqs.as_c(), cout.as_c())
        self.step_wait_compact(slot)
        return cout

    # ---- device path -------------------------------------------------------------------------
    def step_device(self, inbox_c: abi.InboxC, outbox_c: abi.OutboxC, stream: int = 0):
        _check(lib().rafting_step_device(self._h, C.byref(inbox_c), C.byref(outbox_c), C.c_void_p(stream)),
               "rafting_step_device")

    # ---- introspection -----------------------------------------------------------------------
    def export(self, gid: int) -> abi.GroupState:
        st = abi.GroupState()
        _check(lib().rafting_state_export(self._h, gid, C.byref(st)), "rafting_state_export")
        return st

    def export_bulk(self, first: int, count: int):
        arr = (abi.GroupState * count)()
        _check(lib().rafting_state_export_bulk(self._h, first, count, C.cast(arr, C.c_void_p)), "rafting_state_export_bulk")
        return arr

    def digest(self, first: int, count: int) -> np.ndarray:
        out = np.zeros(count, dtype=np.uint64)
        _check(lib().rafting_state_digest(self._h, first, count, out.ctypes.data), "rafting_state_digest")
        return out

    def log_term(self, gid: int, index: int) -> int:
        t = C.c_int64()
        _check(lib().rafting_log_term(self._h, gid, index, C.byref(t)), "rafting_log_term")
        return t.value

    def checkpoint(self):
        _check(lib().rafting_checkpoint(self._h), "rafting_checkpoint")

    def restore(self, sync: bool = True):
        if sync:
            _check(lib().rafting_restore(self._h), "rafting_restore")
        else:
            _check(lib().rafting_restore_async(self._h), "rafting_restore_async")

    def state_save(self, path: str):
        _check(lib().rafting_state_save(self._h, path.encode()), "rafting_state_save")

    def state_load(self, path: str):
        _check(lib().rafting_state_load(self._h, path.encode()), "rafting_state_load")

    def allgather_last(self) -> np.ndarray:
        out = np.zeros(getattr(self, "world", 1) * self.G, dtype=np.int64)
        _check(lib().rafting_allgather_last(self._h, out.ctypes.data), "rafting_allgather_last")
        return out

    def stream(self) -> int:
        s = C.c_void_p()
        _check(lib().rafting_engine_stream(self._h, C.byref(s)), "rafting_engine_stream")
        return s.value or 0

    def counters(self) -> tuple[int, int]:
        a, b = C.c_uint64(), C.c_uint64()
        _check(lib().rafting_engine_counters(self._h, C.byref(a), C.byref(b)), "rafting_engine_counters")
        return a.value, b.value

    # ---- multi-GPU summary ---------------------------------------------------------------------
    def commit_slice(self) -> tuple[int, int]:
        p, n = C.c_void_p(), C.c_uint32()
        _check(lib().rafting_commit_slice(self._h, C.byref(p), C.byref(n)), "rafting_commit_slice")
        return p.value, n.value

    @staticmethod
    def comm_unique_id() -> bytes:
        buf = C.create_string_buffer(128)
        n = C.c_size_t(128)
        _check(lib().rafting_comm_unique_id(buf, C.byref(n)), "rafting_comm_unique_id")
        return buf.raw[:n.value]

    def comm_init(self, rank: int, world: int, uid: bytes | None):
        if uid is None:
            _check(lib().rafting_comm_init(self._h, rank, world, None, 0), "rafting_comm_init")
        else:
            b = C.create_string_buffer(uid, len(uid))
            _check(lib().rafting_comm_init(self._h, rank, world, b, len(uid)), "rafting_comm_init")
        self.rank, self.world = rank, world

    def allgather_commit(self, to_host: bool = True, src: int | None = None):
        """Cross-shard commitIndex summary.  src = device pointer of the column to gather (normally the step's outbox
        commit_index column); None = the live table column."""
        world = getattr(self, "world", 1)
        dev = C.c_void_p()
        if to_host:
            out = np.zeros(world * self.G, dtype=np.int64)
            _check(lib().rafting_allgather_commit_from(self._h, src, out.ctypes.data, C.byref(dev)), "rafting_allgather_commit_from")
            return out
        _check(lib().rafting_allgather_commit_from(self._h, src, None, C.byref(dev)), "rafting_allgather_commit_from")
        return dev.value

    @staticmethod
    def comm_init_all(engines: list["Engine"]):
        """ONE process owning len(engines) shards: engines[r] becomes rank r (grouped ncclCommInitRank)."""
        arr = (C.c_void_p * len(engines))(*[e._h for e in engines])
        _check(lib().rafting_comm_init_all(arr, len(engines)), "rafting_comm_init_all")
        for r, e in enumerate(engines):
            e.rank, e.world = r, len(engines)

    @staticmethod
    def allgather_commit_all(engines: list["Engine"], srcs: list[int] | None = None) -> list[np.ndarray]:
        n = len(engines)
        arr = (C.c_void_p * n)(*[e._h for e in engines])
        outs = [np.zeros(n * e.G, dtype=np.int64) for e in engines]
        ho = (C.c_void_p * n)(*[o.ctypes.data for o in outs])
        sr = None if srcs is None else (C.c_void_p * n)(*srcs)
        _check(lib().rafting_allgather_commit_all(arr, n, sr, ho, None), "rafting_allgather_commit_all")
        return outs

    def step_device_seq(self, ins, outs, n: int, gather: bool = False, stream: int = 0):
        """ins / outs: ctypes arrays of abi.InboxC / abi.OutboxC with device pointers; n steps enqueued by one call."""
        _check(lib().rafting_step_device_seq(self._h, C.cast(ins, C.c_void_p), C.cast(outs, C.c_void_p), n, 1 if gather else 0,
                                             C.c_void_p(stream)), "rafting_step_device_seq")


    # ---- HBM segmented entry buffer (payload side of RaftLog) ------------------------------------
    ENTRY_REF = np.dtype([("gid", "<u4"), ("len", "<u4"), ("index", "<i8"), ("term", "<i8"), ("blob_off", "<u8")])

    def log_config(self, segment_bytes=1 << 18, hbm_segments=64, ring_slots=64):
        _check(lib().rafting_log_config(self._h, segment_bytes, hbm_segments, ring_slots), "rafting_log_config")

    def log_append(self, entries):
        """entries: iterable of (gid, index, term, payload bytes) — RocksLog.newEntry / append (RocksLog.java:82-89,169-196)."""
        entries = list(entries)
        refs = np.zeros(len(entries), dtype=self.ENTRY_REF)
        blob = bytearray()
        for k, (gid, index, term, payload) in enumerate(entries):
            refs[k] = (gid, len(payload), index, term, len(blob))
            blob += payload
            blob += b"\0" * (-len(blob) % 16)
        buf = np.frombuffer(bytes(blob) or b"\0" * 8, dtype=np.uint8)
        _check(lib().rafting_log_append(self._h, refs.ctypes.data, len(refs), buf.ctypes.data, len(blob)), "rafting_log_append")

    def log_read(self, gid, first_index, max_n, blob_cap=1 << 20):
        """RaftLog.batch(first_index, max_n) payload side (RocksLog.java:131-166): [(index, term, bytes)]."""
        refs = np.zeros(max(max_n, 1), dtype=self.ENTRY_REF)
        blob = np.zeros(blob_cap, dtype=np.uint8)
        n = C.c_uint32()
        _check(lib().rafting_log_read(self._h, gid, first_index, max_n, refs.ctypes.data, blob.ctypes.data, blob_cap, C.byref(n)),
               "rafting_log_read")
        return [(int(r["index"]), int(r["term"]), blob[int(r["blob_off"]):int(r["blob_off"]) + int(r["len"])].tobytes())
                for r in refs[:n.value]]

    def log_gather(self, ranges, blob_cap=1 << 24):
        """ranges: [(gid, first, count)] -> [(gid, index, term, bytes | None)] in request order."""
        g = np.array([r[0] for r in ranges], dtype=np.uint32)
        f = np.array([r[1] for r in ranges], dtype=np.int64)
        c = np.array([r[2] for r in ranges], dtype=np.uint32)
        cap = int(c.sum()) + 1
        refs = np.zeros(cap, dtype=self.ENTRY_REF)
        blob = np.zeros(blob_cap, dtype=np.uint8)
        n, nb = C.c_uint32(), C.c_size_t()
        _check(lib().rafting_log_gather(self._h, len(ranges), g.ctypes.data, f.ctypes.data, c.ctypes.data, refs.ctypes.data, cap,
                                        blob.ctypes.data, blob_cap, C.byref(n), C.byref(nb)), "rafting_log_gather")
        return self._gathered(refs[:n.value], blob)

    @staticmethod
    def _gathered(refs, blob) -> list:
        """refs (ENTRY_REF records) + blob -> [(gid, index, term, bytes | None)], as log_gather returns them"""
        out = []
        for r in refs:
            if int(r["len"]) == 0xFFFFFFFF:
                out.append((int(r["gid"]), int(r["index"]), 0, None))
            else:
                out.append((int(r["gid"]), int(r["index"]), int(r["term"]),
                            blob[int(r["blob_off"]):int(r["blob_off"]) + int(r["len"])].tobytes()))
        return out

    def log_gather_step_begin(self, slot: int, refs: np.ndarray, blob: np.ndarray, plans: np.ndarray,
                              refs_cap: int | None = None, blob_cap: int | None = None, plans_cap: int | None = None):
        """rafting_log_gather_step_begin: gather, on the entry buffer's stream, the payloads of the AppendEntries plans of the
        compact step last waited for in `slot`.  refs (ENTRY_REF), blob (uint8) and plans (abi.PLAN_REF) receive them; pinned
        arrays are written by the device directly.  They must stay alive until log_gather_step_wait."""
        for a, dt in ((refs, self.ENTRY_REF), (blob, np.dtype(np.uint8)), (plans, abi.PLAN_REF)):
            if a.dtype != dt or not a.flags.c_contiguous:
                raise TypeError(f"expected a contiguous {dt} array")
        rc = len(refs) if refs_cap is None else refs_cap
        bc = len(blob) if blob_cap is None else blob_cap
        pc = len(plans) if plans_cap is None else plans_cap
        if rc > len(refs) or bc > len(blob) or pc > len(plans):
            raise ValueError("a cap beyond its buffer")
        _check(lib().rafting_log_gather_step_begin(self._h, slot, refs.ctypes.data if len(refs) else None, rc,
                                                   blob.ctypes.data if len(blob) else None, bc,
                                                   plans.ctypes.data if len(plans) else None, pc), "rafting_log_gather_step_begin")

    def log_gather_step_wait(self, slot: int) -> tuple[int, int, int, int]:
        """-> (n_refs, bytes, n_plans, host_served).  A cap that was too small raises RaftingError (E_CAPACITY) whose `sizes`
        holds the same tuple, with the sizes needed."""
        n, b, p, h = C.c_uint32(), C.c_size_t(), C.c_uint32(), C.c_uint32()
        rc = lib().rafting_log_gather_step_wait(self._h, slot, C.byref(n), C.byref(b), C.byref(p), C.byref(h))
        sizes = (n.value, b.value, p.value, h.value)
        if rc:
            ex = RaftingError(rc, "rafting_log_gather_step_wait")
            ex.sizes = sizes
            raise ex
        return sizes

    def log_gather_step(self, slot: int = 0, refs_cap: int = 1 << 16, blob_cap: int = 1 << 24, plans_cap: int = 1 << 16):
        """Synchronous: -> ([(gid, index, term, bytes | None)] as log_gather returns them, plan records (abi.PLAN_REF),
        host_served).  Grows the buffers and gathers again when a cap was too small."""
        while True:
            refs = np.zeros(refs_cap, dtype=self.ENTRY_REF)
            blob = np.zeros(blob_cap, dtype=np.uint8)
            plans = np.zeros(plans_cap, dtype=abi.PLAN_REF)
            self.log_gather_step_begin(slot, refs, blob, plans)
            try:
                n, _, p, h = self.log_gather_step_wait(slot)
            except RaftingError as ex:
                if ex.rc != -5:
                    raise
                n, b, p, _ = ex.sizes
                refs_cap, blob_cap, plans_cap = max(refs_cap, n), max(blob_cap, b), max(plans_cap, p)
                continue
            return self._gathered(refs[:n], blob), plans[:p].copy(), h

    GATHER_TICKETS = 4

    def log_gather_begin(self, ticket: int, ranges, refs: np.ndarray, blob: np.ndarray,
                         refs_cap: int | None = None, blob_cap: int | None = None):
        """rafting_log_gather_begin: gather, on the entry buffer's stream, the payloads of `ranges` ([(gid, first, count)], or a
        (gids, firsts, counts) tuple of arrays) under `ticket`.  refs (ENTRY_REF) and blob (uint8) receive what log_gather
        would return; pinned arrays are written by the device directly.  They must stay alive until log_gather_wait."""
        for a, dt in ((refs, self.ENTRY_REF), (blob, np.dtype(np.uint8))):
            if a.dtype != dt or not a.flags.c_contiguous:
                raise TypeError(f"expected a contiguous {dt} array")
        if isinstance(ranges, tuple):
            g, f, c = (np.ascontiguousarray(x, dt) for x, dt in zip(ranges, (np.uint32, np.int64, np.uint32)))
        else:
            r = list(ranges)
            g = np.array([x[0] for x in r], dtype=np.uint32)
            f = np.array([x[1] for x in r], dtype=np.int64)
            c = np.array([x[2] for x in r], dtype=np.uint32)
        rc = len(refs) if refs_cap is None else refs_cap
        bc = len(blob) if blob_cap is None else blob_cap
        if rc > len(refs) or bc > len(blob):
            raise ValueError("a cap beyond its buffer")
        n = len(g)
        _check(lib().rafting_log_gather_begin(self._h, ticket, n, g.ctypes.data if n else None, f.ctypes.data if n else None,
                                              c.ctypes.data if n else None, refs.ctypes.data if len(refs) else None, rc,
                                              blob.ctypes.data if len(blob) else None, bc), "rafting_log_gather_begin")

    def log_gather_wait(self, ticket: int) -> tuple[int, int, int]:
        """-> (n_refs, bytes, host_served).  A blob that was too small raises RaftingError (E_CAPACITY) whose `sizes` holds the
        same tuple, with the bytes needed."""
        n, b, h = C.c_uint32(), C.c_size_t(), C.c_uint32()
        rc = lib().rafting_log_gather_wait(self._h, ticket, C.byref(n), C.byref(b), C.byref(h))
        sizes = (n.value, b.value, h.value)
        if rc:
            ex = RaftingError(rc, "rafting_log_gather_wait")
            ex.sizes = sizes
            raise ex
        return sizes

    def log_stats(self) -> dict:
        v = np.zeros(11, dtype=np.uint64)
        lib().rafting_log_stats(self._h, v.ctypes.data, 11)
        return dict(zip(("appended", "head", "spilled_bytes", "hbm_hits", "cold_hits", "indexed", "gather_kernel_ns",
                         "gather_bytes", "trimmed", "cold_freed_bytes", "spills_skipped"), v.tolist()))

    def log_trim(self, first_gid: int = 0, count: int | None = None) -> tuple[int, int]:
        """GC behind RaftLog.flush: (index entries dropped, cold bytes freed)."""
        d, f = C.c_uint64(), C.c_uint64()
        _check(lib().rafting_log_trim(self._h, first_gid, self.G - first_gid if count is None else count, C.byref(d), C.byref(f)),
               "rafting_log_trim")
        return d.value, f.value

    # ---- durable tier of the entry buffer (what flushWal(true) gives RocksLog) -------------------------------------------
    def log_store_open(self, path: str, cold_max_segments: int = 0) -> int:
        """Opens (creates) the entry file and replays it; returns the number of records recovered."""
        n = C.c_uint64()
        _check(lib().rafting_log_store_open(self._h, path.encode(), cold_max_segments, C.byref(n)), "rafting_log_store_open")
        return n.value

    def log_sync(self):
        _check(lib().rafting_log_sync(self._h), "rafting_log_sync")

    def log_mark(self, gid: int, lo: int, hi: int, epoch_index: int, epoch_term: int):
        _check(lib().rafting_log_mark(self._h, gid, lo, hi, epoch_index, epoch_term), "rafting_log_mark")

    def log_recovered(self, gid: int):
        """-> (abi.GroupInit with epoch / key range / last term, [(first index, term), ...] runs oldest first)"""
        gi = abi.GroupInit()
        runs = np.zeros((64, 2), dtype=np.int64)
        n = C.c_uint32()
        _check(lib().rafting_log_recovered(self._h, gid, C.byref(gi), runs.ctypes.data, 64, C.byref(n)), "rafting_log_recovered")
        return gi, [tuple(int(x) for x in r) for r in runs[:n.value]]

    def log_export_kv(self, gid: int, index: int, cap: int = 1 << 16) -> tuple[bytes, bytes]:
        key, val, n = C.create_string_buffer(8), C.create_string_buffer(cap), C.c_size_t()
        _check(lib().rafting_log_export_kv(self._h, gid, index, key, val, cap, C.byref(n)), "rafting_log_export_kv")
        return key.raw, val.raw[:n.value]

    def log_store_stats(self) -> dict:
        a = (C.c_uint64 * 6)()
        _check(lib().rafting_log_store_stats(self._h, C.byref(a)), "rafting_log_store_stats")
        return dict(zip(("file_bytes", "synced_bytes", "syncs", "file_hits", "cold_evicted", "cold_resident"), list(a)))

    def allgather_join(self):
        _check(lib().rafting_allgather_join(self._h), "rafting_allgather_join")


class Lease:
    """Pinned host staging for one step (rafting_lease_t): numpy views over the engine's buffers."""

    IN_OPS = (("op_meta", np.uint64), ("op_nr", abi.I64X2), ("op_ab", abi.I64X2), ("op_cd", abi.I64X2), ("op_e", np.int64))
    IN_EVS = (("ev_meta", np.uint64), ("ev_tn", abi.I64X2), ("ev_el", abi.I64X2))

    def __init__(self, eng: Engine, lc: abi.LeaseC, rows: int, n: int, gcols: int | None = None):
        self.eng, self.c, self.rows, self.n = eng, lc, rows, n
        F, G = eng.F, (eng.G if gcols is None else gcols)
        i = lc.inbox
        self._orig = {name: getattr(i, name) for name, _ in self.IN_OPS + self.IN_EVS}
        self._orig["row_now"] = i.row_now
        self.gids = _np_view(i.gids, np.uint32, (i.n_active,)) if i.n_active else None
        self.row_now = _np_view(i.row_now, np.int64, (rows,))
        for name, dt in self.IN_OPS:
            setattr(self, name, _np_view(getattr(i, name), dt, (rows, n)))
        self.ent_terms = _np_view(i.ent_terms, np.int64, (max(i.ent_count, 1),))
        for name, dt in self.IN_EVS:
            setattr(self, name, _np_view(getattr(i, name), dt, (rows, n, F)))
        o = lc.outbox
        self.out = abi.Outbox.__new__(abi.Outbox)
        self.out.rows, self.out.n, self.out.F, self.out.G = rows, n, F, G
        for name, dt, lane in abi.Outbox.ROW_COLS:
            shape = (rows, n, F) if lane else (rows, n)
            setattr(self.out, name, _np_view(getattr(o, name), dt, shape))
        for name, dt in abi.Outbox.GROUP_COLS:
            setattr(self.out, name, _np_view(getattr(o, name), dt, (G,)))

    def use(self, ops: bool = True, events: bool = True, flags: int = 0):
        """Declare which column families this step carries (absent ones are neither copied nor read)."""
        i = self.c.inbox
        for name, _ in self.IN_OPS:
            setattr(i, name, self._orig[name] if ops else None)
        for name, _ in self.IN_EVS:
            setattr(i, name, self._orig[name] if events else None)
        i.flags = flags
        self._ops = ops

    def fill_from(self, ib: abi.Inbox):
        if ib.gids is not None:
            self.gids[:] = ib.gids
        self.c.inbox.rows = ib.rows
        if ib.row_now is not None:
            self.row_now[:ib.rows] = ib.row_now
        else:
            self.row_now[:] = 0
        self.use(ops=ib.op_meta is not None, events=ib.ev_meta is not None, flags=ib.flags)
        if ib.op_meta is not None:
            for name, _ in self.IN_OPS:
                col = getattr(ib, name)
                if col is None:                      # e.g. op_cd / op_e absent in a NO_REQUESTS step
                    setattr(self.c.inbox, name, None)
                else:
                    getattr(self, name)[:ib.rows] = col
        if ib.ent_count:
            self.ent_terms[:ib.ent_count] = ib.ent_terms[:ib.ent_count]
        self.c.inbox.ent_count = ib.ent_count
        if ib.ev_meta is not None:
            for name, _ in self.IN_EVS:
                getattr(self, name)[:ib.rows] = getattr(ib, name)

    def run(self):
        _check(lib().rafting_step(self.eng._h, C.byref(self.c)), "rafting_step")

    def begin(self):
        _check(lib().rafting_step_begin(self.eng._h, C.byref(self.c)), "rafting_step_begin")

    def wait(self):
        _check(lib().rafting_step_wait(self.eng._h, C.byref(self.c)), "rafting_step_wait")

    def release(self):
        """Give back a lease that will not be stepped."""
        _check(lib().rafting_lease_release(self.eng._h, C.byref(self.c)), "rafting_lease_release")

    def outbox_copy(self) -> abi.Outbox:
        o = abi.Outbox.__new__(abi.Outbox)
        o.rows, o.n, o.F, o.G = self.out.rows, self.out.n, self.out.F, self.out.G
        rows = self.c.inbox.rows
        sweep = bool(self.row_now[:rows].any())
        for name, _, _ in abi.Outbox.ROW_COLS:
            col = getattr(self.out, name)[:rows].copy()
            # without group ops (and without a sweep) the engine neither produces nor copies back the
            # reply / plan families: they read as "nothing" (zero meta)
            if not (getattr(self, "_ops", True) or sweep) and name in ("rep_meta", "plan_meta"):
                col[...] = 0
            setattr(o, name, col)
        o.rows = rows
        for name, _ in abi.Outbox.GROUP_COLS:
            setattr(o, name, getattr(self.out, name).copy())
        return o
