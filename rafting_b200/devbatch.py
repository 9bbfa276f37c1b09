"""HBM-resident batches for the device path (rafting_step_device): torch is used ONLY to own device
memory and streams; the columns are raw bytes whose addresses go into the C structs."""
from __future__ import annotations

import torch

from . import abi

_IN_COLS = (("op_meta", 8, False), ("op_nr", 16, False), ("op_ab", 16, False), ("op_cd", 16, False), ("op_e", 8, False),
            ("ev_meta", 8, True), ("ev_tn", 16, True), ("ev_el", 16, True))
_OUT_ROW = (("rep_meta", 4, False), ("rep_term", 8, False), ("plan_meta", 8, True), ("plan_pp", 16, True),
            ("plan_lc", 16, True), ("plan_epoch", 8, True), ("ballot_meta", 8, False), ("ballot_term", 8, False),
            ("ballot_last", 16, False))
_OUT_GRP = (("commit_index", 8), ("current_term", 8), ("role_word", 4), ("incarnation", 4), ("err_word", 4), ("last_entry", 16))


class DevInbox:
    def __init__(self, rows, n, F, device, requests=False, unavail=True):
        """requests=False omits op_cd/op_e (no inbound-request ops); unavail=False also omits op_ab (its only use in
        such a step is the unavailable-follower mask of SUBMIT / TIMEOUT: absent == nobody unavailable)."""
        self.rows, self.n, self.F = rows, n, F
        self.t = {}
        for name, sz, lane in _IN_COLS:
            if not requests and name in ("op_cd", "op_e"):
                continue
            if not unavail and name == "op_ab":
                continue
            cnt = rows * n * (F if lane else 1)
            self.t[name] = torch.zeros(cnt * sz, dtype=torch.uint8, device=device)
        self.flags = 0 if requests else abi.INBOX_NO_REQUESTS
        self.gids = self.row_now = self.ent_terms = None
        self.ent_count = 0

    @classmethod
    def from_host(cls, ib: abi.Inbox, device) -> "DevInbox":
        """Device-resident copy of a host inbox: every column, the active list, the sweep times and the entry pool
        (columns absent on the host stay absent)."""
        import numpy as np

        def dev(a):
            return None if a is None else torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).reshape(-1)).to(device)
        self = cls.__new__(cls)
        self.rows, self.n, self.F = ib.rows, ib.n, ib.F
        self.t = {}
        for name, _, _ in _IN_COLS:
            col = getattr(ib, name)
            if col is not None:
                self.t[name] = dev(col)
        self.flags = ib.flags
        self.gids, self.row_now, self.ent_terms = dev(ib.gids), dev(ib.row_now), dev(ib.ent_terms)
        self.ent_count = ib.ent_count
        return self

    def nbytes(self):
        return sum(t.numel() for t in self.t.values())

    def as_c(self) -> abi.InboxC:
        c = abi.InboxC()
        c.rows, c.n_active = self.rows, 0 if self.gids is None else self.n
        for name, _, _ in _IN_COLS:
            setattr(c, name, self.t[name].data_ptr() if name in self.t else None)
        for name in ("gids", "row_now", "ent_terms"):
            a = getattr(self, name)
            setattr(c, name, None if a is None else a.data_ptr())
        c.ent_count = self.ent_count
        c.flags = self.flags
        return c


class DevOutbox:
    def __init__(self, rows, n, F, G, device, fill=0):
        """G: entries of a per-group column (max_groups, or n_active under RAFTING_INBOX_COMPACT_GROUPS).  Every byte
        starts as `fill`, so a cell the step leaves unwritten keeps it."""
        self.rows, self.n, self.F, self.G = rows, n, F, G
        self.t = {}
        for name, sz, lane in _OUT_ROW:
            self.t[name] = torch.full((rows * n * (F if lane else 1) * sz,), fill, dtype=torch.uint8, device=device)
        for name, sz in _OUT_GRP:
            self.t[name] = torch.full((G * sz,), fill, dtype=torch.uint8, device=device)

    def nbytes(self):
        return sum(t.numel() for t in self.t.values())

    def as_c(self) -> abi.OutboxC:
        c = abi.OutboxC()
        for name in self.t:
            setattr(c, name, self.t[name].data_ptr())
        return c

    def to_host(self) -> abi.Outbox:
        import numpy as np
        o = abi.Outbox(self.rows, self.n, self.F, self.G)
        for name, t in self.t.items():
            a = getattr(o, name)
            a[...] = np.frombuffer(t.cpu().numpy().tobytes(), dtype=a.dtype).reshape(a.shape)
        return o
