"""ctypes binding of the CPU oracle (oracle/raft_oracle.c).  TEST INFRASTRUCTURE ONLY.

Importable from tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference
legs; nothing under rafting_b200/ may import this module.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

from rafting_b200 import abi

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "_build", "liboracle.so")
_lib = None


def build(force: bool = False) -> str:
    src = [os.path.join(_HERE, f) for f in ("raft_oracle.c", "raft_oracle.h")] + \
          [os.path.join(_HERE, "..", "include", "rafting_b200.h")]
    stale = force or not os.path.exists(_LIB_PATH) or any(
        os.path.getmtime(s) > os.path.getmtime(_LIB_PATH) for s in src)
    if stale:
        subprocess.check_call(["make", "-C", _HERE, "-s"])
    return _LIB_PATH


def lib():
    global _lib
    if _lib is None:
        build()
        L = C.CDLL(_LIB_PATH)
        L.orc_create.restype = C.c_void_p
        L.orc_create.argtypes = [C.POINTER(abi.Cfg)]
        L.orc_destroy.argtypes = [C.c_void_p]
        L.orc_group_open.argtypes = [C.c_void_p, C.c_uint32, C.POINTER(abi.GroupInit)]
        L.orc_group_open_bulk.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p]
        L.orc_group_close.argtypes = [C.c_void_p, C.c_uint32]
        L.orc_group_load_runs.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32]
        L.orc_step.argtypes = [C.c_void_p, C.POINTER(abi.InboxC), C.POINTER(abi.OutboxC), C.c_int]
        L.orc_state_export.argtypes = [C.c_void_p, C.c_uint32, C.POINTER(abi.GroupState)]
        L.orc_log_term.argtypes = [C.c_void_p, C.c_uint32, C.c_int64, C.POINTER(C.c_int64)]
        L.orc_events_processed.restype = C.c_uint64
        L.orc_events_processed.argtypes = [C.c_void_p]
        L.orc_major_indices.argtypes = [C.POINTER(C.c_int64), C.c_int, C.POINTER(C.c_int64)]
        L.orc_state_apply.argtypes = [C.POINTER(C.c_int64), C.c_int, C.POINTER(C.c_int64), C.POINTER(C.c_int64)]
        L.orc_backoff_step.restype = C.c_int64
        L.orc_backoff_step.argtypes = [C.c_int32]
        L.orc_is_better.restype = C.c_int
        L.orc_is_better.argtypes = [C.c_int, C.c_int64, C.c_int, C.c_int, C.c_int64, C.c_int, C.c_int]
        L.orc_draw.restype = C.c_int64
        L.orc_draw.argtypes = [C.c_uint64, C.c_uint32, C.c_uint32, C.c_int64]
        _lib = L
    return _lib


class Oracle:
    """Same surface as rafting_b200.engine.Engine so a test can drive both with one script."""

    def __init__(self, cfg: abi.Cfg):
        self.cfg = cfg
        self.F = cfg.replicas - 1
        self.G = cfg.max_groups
        self._h = lib().orc_create(C.byref(cfg))
        if not self._h:
            raise ValueError("orc_create failed (bad cfg)")

    def close(self):
        if self._h:
            lib().orc_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def open_group(self, gid: int, **kw):
        gi = group_init(**kw)
        rc = lib().orc_group_open(self._h, gid, C.byref(gi))
        if rc:
            raise ValueError(f"orc_group_open rc={rc}")

    def open_bulk(self, first_gid: int, inits: np.ndarray):
        inits = np.ascontiguousarray(inits, dtype=abi.GROUP_INIT_DTYPE)
        rc = lib().orc_group_open_bulk(self._h, first_gid, len(inits), inits.ctypes.data)
        if rc:
            raise ValueError(f"orc_group_open_bulk rc={rc}")

    def load_runs(self, gid: int, runs):
        a = np.array(runs, dtype=np.int64).reshape(-1, 2)
        rc = lib().orc_group_load_runs(self._h, gid, a.ctypes.data, len(a))
        if rc:
            raise ValueError(f"orc_group_load_runs rc={rc}")

    def close_group(self, gid: int):
        lib().orc_group_close(self._h, gid)

    def step(self, inbox: abi.Inbox, threads: int = 1, out: abi.Outbox | None = None) -> abi.Outbox:
        """out: a caller-owned outbox to step into (cells the step does not write keep their bytes); None: a fresh
        zeroed one."""
        n = inbox.n
        compact = inbox.gids is not None and (inbox.flags & abi.INBOX_COMPACT_GROUPS)
        if out is None:
            out = abi.Outbox(inbox.rows, n, self.F, n if compact else self.G)
        elif (out.rows, out.n, out.F, out.G) != (inbox.rows, n, self.F, n if compact else self.G):
            raise ValueError("outbox shape does not match the inbox")
        ic, oc = inbox.as_c(), out.as_c()
        rc = lib().orc_step(self._h, C.byref(ic), C.byref(oc), threads)
        if rc:
            raise RuntimeError(f"orc_step rc={rc}")
        return out

    def export(self, gid: int) -> abi.GroupState:
        st = abi.GroupState()
        rc = lib().orc_state_export(self._h, gid, C.byref(st))
        if rc:
            raise RuntimeError(f"orc_state_export rc={rc}")
        return st

    def log_term(self, gid: int, index: int) -> int:
        t = C.c_int64()
        lib().orc_log_term(self._h, gid, index, C.byref(t))
        return t.value

    def events(self) -> int:
        return lib().orc_events_processed(self._h)


def group_init(term=0, ballot=-1, epoch_index=0, epoch_term=0, first_index=1, last_index=0, last_term=0,
               commit_index=0, now_ms=0, rand_ms=1000) -> abi.GroupInit:
    gi = abi.GroupInit()
    gi.term, gi.ballot = term, ballot
    gi.epoch_index, gi.epoch_term = epoch_index, epoch_term
    gi.first_index, gi.last_index, gi.last_term = first_index, last_index, last_term
    gi.commit_index, gi.now_ms, gi.rand_ms = commit_index, now_ms, rand_ms
    return gi


def major_indices(match) -> tuple[int, int]:
    arr = (C.c_int64 * len(match))(*match)
    out = (C.c_int64 * 2)()
    lib().orc_major_indices(arr, len(match), out)
    return out[0], out[1]
