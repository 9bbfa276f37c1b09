"""Python restatement of the engine's kernel dispatch (launch_step, rafting_b200/csrc/engine.cu:321-356) and of the
class that classify_kernel gives each position of a class-sorted step (rafting_b200/csrc/step_kernel.cuh:124-162).

The parity matrix of tests/test_engine_gpu.py is checked against `kernels` on the CPU, so a launch the engine can make
without a GPU test behind it fails there; `classes` lets a fuzz case check that it fills every class it is meant to."""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np

from rafting_b200 import abi

SORT_MIN_N = 2048          # engine.cu:328
NCLS = 4                   # step_kernel.cuh:122
CLS_FOLLOWER, CLS_CANDIDATE, CLS_SLOW_LEADER, CLS_STEADY_LEADER = range(NCLS)


def class_sorted(R: int, n: int, flags: int = 0, has_ops: bool = True) -> bool:
    """engine.cu:328: a step that may carry requests, with ops, n >= 2048 and F <= 8 is launched class-sorted."""
    return not (flags & abi.INBOX_NO_REQUESTS) and has_ops and n >= SORT_MIN_N and R - 1 <= 8


def kernels(R: int, n: int, flags: int = 0, has_ops: bool = True, fix: bool = False) -> tuple[tuple[str, ...], str]:
    """(kernels launched, in launch order; mode) for one step of n positions at R replicas.  fix: the engine has cfg.flags
    set, so the step and slow kernels are the FIX instantiations (named with a trailing ",true"), and at R = 3 only a step
    that promises no inbound request runs in pair_kernel (engine.cu, launch_step_t)."""
    F = R - 1
    srt = class_sorted(R, n, flags, has_ops)
    t = ",true" if fix else ""
    ks = []
    if srt:
        ks.append("classify_kernel")                                       # engine.cu:329-331
        if 2 <= F <= 4:
            ks.append(f"slow_kernel<2,4{t}>" if F == 2 else f"slow_kernel<4,4{t}>")   # engine.cu:334-339
    if F == 1:
        ft, main = 1, f"step_kernel<1,3{t}>"                               # engine.cu:340
    elif F == 2:
        pair = not srt and (not fix or bool(flags & abi.INBOX_NO_REQUESTS))
        ft, main = 2, ("pair_kernel" if pair else f"step_kernel<2,3{t}>")  # engine.cu:344-348
    elif F <= 4:
        ft, main = 4, f"step_kernel<4,3{t}>"                               # engine.cu:349
    elif F <= 8:
        ft, main = 8, f"step_kernel<8,2{t}>"                               # engine.cu:350
    else:
        ft, main = 32, f"looped::step_kernel<32,0{t}>"                     # engine.cu:351
    ks.append(main)
    if srt and not 2 <= F <= 4:
        ks.append(f"slow_group<{ft}>")        # the slow classes run inside the step kernel (step_body.inc:414-418)
    return tuple(ks), "class-sorted" if srt else "unsorted"


@dataclass(frozen=True)
class SeqLaunch:
    """One launch of a rafting_step_device_seq call: its kernels and mode (as `kernels`), whether pair_kernel is launched
    programmatically (Hopper PDL: its blocks start, and stage their first inbox rows, before the launch ahead of it on the
    stream has finished), and the kernels of that launch (None for the first launch of the call)."""
    kernels: tuple[str, ...]
    mode: str
    programmatic: bool
    after: tuple[str, ...] | None

    @property
    def predecessor(self) -> str | None:
        """The kernel that runs directly ahead of this launch's first kernel on the stream."""
        return None if self.after is None else self.after[-1]


def sequence(R: int, inboxes, gather: bool = False, fix: bool = False) -> list[SeqLaunch]:
    """The launches of one rafting_step_device_seq call over `inboxes` (engine.cu): launch k > 0 of a call without gathers
    follows launch k-1's last kernel directly, and when its main kernel is pair_kernel it is launched programmatically.
    With gathers every launch waits behind a copy of the commit column instead, and none is."""
    out, prev = [], None
    for k, ib in enumerate(inboxes):
        ks, mode = kernels(R, ib.n, ib.flags, ib.op_meta is not None, fix)
        out.append(SeqLaunch(ks, mode, k > 0 and not gather and ks[-1] == "pair_kernel", prev))
        prev = ks
    return out


def reachable() -> set[tuple[tuple[str, ...], str]]:
    """Every (kernels, mode) a step can take, over R = 2..33 and both sides of the sort threshold."""
    out = set()
    for R in range(2, abi.MAX_REPLICAS + 1):
        for n in (SORT_MIN_N - 1, SORT_MIN_N):
            for flags in (0, abi.INBOX_NO_REQUESTS):
                out.add(kernels(R, n, flags))
    return out


def classes(ref, ib: abi.Inbox) -> np.ndarray:
    """classify_kernel's class of every position of `ib`, from `ref`'s exported state before the step."""
    G = ref.cfg.max_groups
    cls = np.empty(ib.n, dtype=np.int8)
    sweep = ib.row_now if ib.row_now is not None else np.zeros(ib.rows, dtype=np.int64)
    for i in range(ib.n):
        gid = int(ib.gids[i]) if ib.gids is not None else i
        if gid >= G:
            cls[i] = CLS_SLOW_LEADER
            continue
        st = ref.export(gid)
        if st.role == abi.ROLE_FOLLOWER:
            cls[i] = CLS_FOLLOWER
        elif st.role == abi.ROLE_CANDIDATE:
            cls[i] = CLS_CANDIDATE
        else:
            slow = not (st.alive and st.leader_prepared)
            if not slow and ib.op_meta is not None:
                slow = any(sweep[r] == 0 and (int(ib.op_meta[r, i]) & 0xFF) > abi.OP_TIMEOUT for r in range(ib.rows))
            cls[i] = CLS_SLOW_LEADER if slow else CLS_STEADY_LEADER
    return cls
