"""Shared drivers for the parity tests: one script drives the CPU oracle and the CUDA engine
through the identical batch interface and compares outboxes and exported state byte for byte."""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass, field

import numpy as np

from rafting_b200 import abi, workload
from rafting_b200.abi import (EV_AE_ACK, EV_IS_ACK, EV_PV_REPLY, EV_RV_REPLY, OUT_CANCELED, OUT_ERROR, OUT_OK,
                              ROLE_CANDIDATE, ROLE_FOLLOWER, ROLE_LEADER)

T0 = workload.T0_MS


def state_bytes(st: abi.GroupState, F: int) -> bytes:
    used = abi.GroupState.followers.offset + C.sizeof(abi.FollowerState) * F
    return bytes(st)[:used]


def assert_states_equal(a, b, gids, F, where=""):
    for gid in gids:
        sa, sb = a.export(gid), b.export(gid)
        if state_bytes(sa, F) != state_bytes(sb, F):
            da, db = sa.as_dict(), sb.as_dict()
            diff = {k: (da[k], db[k]) for k in da if da[k] != db[k]}
            raise AssertionError(f"group {gid} state differs {where}: {diff}")


def assert_outbox_equal(oa: abi.Outbox, ob: abi.Outbox, gids=None, where=""):
    bad = oa.equal(ob, gids)
    if bad:
        name = bad[0]
        a, b = getattr(oa, name), getattr(ob, name)
        if a.shape == b.shape:
            idx = np.argwhere(a != b)[:5].tolist()
        else:
            idx = "shape"
        raise AssertionError(f"outbox column(s) {bad} differ {where}; first diffs of {name} at {idx}")


def init_array(n, terms=None, **common) -> np.ndarray:
    a = np.zeros(n, dtype=abi.GROUP_INIT_DTYPE)
    a["ballot"] = -1
    a["first_index"] = 1
    a["now_ms"] = T0 - 2000
    a["rand_ms"] = 0
    for k, v in common.items():
        a[k] = v
    if terms is not None:
        a["term"] = terms
    return a


def elect_all(sut, w1: workload.WlCfg):
    """Follower -> PreVote round -> Candidate -> Leader for every group, unanimous grants."""
    out = None
    phases = (0, 1, 2) if sut.cfg.pre_vote else (0, 2)
    for ph in phases:
        ib = workload.election_inbox_host(w1, ph, out)
        out = sut.step(ib)
    return out


def run_leader_workload(suts, w: workload.WlCfg, steps: int, compare=True, first_step=0, prevs=None, drop_ab=False):
    """Drives every SUT in `suts` with the SAME stream, generated from the FIRST sut's outbox
    (after checking the others produced the identical outbox).  Returns the last outboxes."""
    prev = prevs
    for k in range(first_step, first_step + steps):
        ib = workload.leader_inbox_host(w, k, prev)
        if drop_ab:
            ib.op_ab = None          # nobody unavailable: the column is simply absent
        outs = [s.step(ib) for s in suts]
        if compare:
            for o in outs[1:]:
                assert_outbox_equal(outs[0], o, where=f"at step {k}")
        prev = outs[0]
    return prev


# ---------------------------------------------------------------------------------------------
# random fuzz over every op / event kind, steered by the reference SUT's exported state
# ---------------------------------------------------------------------------------------------
class Fuzzer:
    """Knobs, all off by default (off, every random draw is the one the plain fuzz makes):
      gids            an active list, strictly increasing, that may end in ids >= max_groups; position i drives gids[i]
      leader_share    that fraction of the positions gets only SUBMIT / TIMEOUT ops and in-term replies, so that
                      groups elected beforehand (elect_all) stay steady-state leaders
      sweep_every     every k-th row of the stream is a timer sweep row (row_now set), ops and lane events kept
      stray_requests  every k-th step is flagged RAFTING_INBOX_NO_REQUESTS and keeps its requests
      t0              added to every time the fuzz writes
      jump            added to the time at a third and at two thirds of every row, so that the row's last third lies more
                      than 2 * jump ms after its first position
      unavail_lanes   SUBMIT / TIMEOUT draw their unavailable mask from that many low bits (default 2)
      near_commit     an inbound AppendEntries carries a leader commit a few entries above its prevLogIndex and the
                      group's own commit index, instead of one drawn from [0, last + 3), and most carry no election-timeout
                      draw: with logs near 2^40 they then fit a compact request record (d_commit an int32, no draw)"""

    def __init__(self, cfg: abi.Cfg, ref, seed=1, rows=3, n=None, gids=None, leader_share=0.0, sweep_every=0,
                 stray_requests=0, t0=0, jump=0, unavail_lanes=2, near_commit=False):
        self.cfg, self.ref = cfg, ref
        self.rng = np.random.default_rng(seed)
        self.aux = np.random.default_rng([seed, 0xA5])     # the knobs draw from here, never from rng
        self.rows = rows
        self.gids = None if gids is None else np.ascontiguousarray(gids, dtype=np.uint32)
        if self.gids is not None:
            assert (np.diff(self.gids.astype(np.int64)) > 0).all(), "active list must be strictly increasing"
        self.n = len(self.gids) if self.gids is not None else (n or cfg.max_groups)
        self.F = cfg.replicas - 1
        self.now = T0 + t0
        self.pending = {}      # position -> list of (lane, kind, inc, epoch, last) replies owed to the SUT
        self.steady = np.zeros(self.n, dtype=bool)
        if leader_share:
            self.steady[self.aux.permutation(self.n)[:int(leader_share * self.n)]] = True
        self.sweep_every, self.stray = sweep_every, stray_requests
        self.jump, self.unavail, self.near_commit = jump, 1 << unavail_lanes, near_commit
        self.row_count = self.step_count = 0

    def gid(self, i: int) -> int:
        return int(self.gids[i]) if self.gids is not None else i

    def _peer(self):
        R = self.cfg.replicas
        s = int(self.rng.integers(0, R - 1))
        return s if s < self.cfg.local_slot else s + 1

    def make(self, last_out: abi.Outbox | None) -> abi.Inbox:
        rng, F, G = self.rng, self.F, self.cfg.max_groups
        ib = abi.Inbox(self.rows, self.n, F, ent_cap=self.rows * self.n * 8, gids=self.gids, sweep=self.sweep_every > 0)
        self.step_count += 1
        if self.stray and self.step_count % self.stray == 0:
            ib.flags |= abi.INBOX_NO_REQUESTS
        # harvest reply obligations from the last outbox (a position outside the table has no written cells)
        if last_out is not None:
            for r in range(last_out.rows):
                for i in range(self.n):
                    if self.gid(i) >= G:
                        continue
                    for f in range(F):
                        pm = int(last_out.plan_meta[r, i, f])
                        k = pm & 0xF
                        if k in (abi.PLAN_AE, abi.PLAN_IS):
                            self.pending.setdefault(i, []).append(
                                (f, EV_IS_ACK if k == abi.PLAN_IS else EV_AE_ACK, pm >> 32,
                                 int(last_out.plan_epoch[r, i, f]), int(last_out.plan_lc[r, i, f]["x"])))
                    bm = int(last_out.ballot_meta[r, i])
                    if bm & 0xF:
                        kind = EV_PV_REPLY if (bm & 0xF) == abi.BALLOT_PREVOTE else EV_RV_REPLY
                        for f in range(F):
                            self.pending.setdefault(i, []).append((f, kind, bm >> 32, 0, 0))
        for r in range(self.rows):
            if self.sweep_every:
                self.row_count += 1
                if self.row_count % self.sweep_every == 0:
                    ib.row_now[r] = self.now + 1
            for i in range(self.n):
                self.now += 1
                if self.jump and i in (self.n // 3, 2 * self.n // 3):
                    self.now += self.jump
                gid = self.gid(i)
                if gid >= G:               # takes no part in the step; neither side writes its cells
                    ib.timeout(r, i, self.now)
                    ib.ack(r, i, 0, self.now, 1, 1, True, 0, 0)
                    continue
                st = self.ref.export(gid)
                if self.steady[i]:
                    self._steady(ib, r, i, st)
                    continue
                term, role = st.current_term, st.role
                u = rng.random()
                if u < 0.25:
                    pass
                elif u < 0.40:
                    ib.submit(r, i, self.now, count=int(rng.integers(1, 4)), unavail=int(rng.integers(0, self.unavail)) if rng.random() < 0.1 else 0)
                elif u < 0.55:
                    ib.timeout(r, i, self.now, rand=int(rng.integers(900, 1801)) if rng.random() < 0.7 else 0,
                               unavail=int(rng.integers(0, self.unavail)) if rng.random() < 0.1 else 0)
                elif u < 0.75:
                    # inbound AppendEntries from a plausible leader
                    t = term + int(rng.choice([-1, 0, 0, 0, 1, 2]))
                    if t < 0:
                        t = 0
                    has = st.last_index >= st.first_index
                    last = st.last_index if has else st.epoch_index
                    mode = rng.random()
                    if mode < 0.6:       # append right after our last entry
                        prev = last
                        prev_t = (st.last_term if has else st.epoch_term)
                    elif mode < 0.8 and last > st.epoch_index + 1:   # overlap: rewrite the tail
                        prev = int(rng.integers(st.epoch_index + 1, last))
                        prev_t = self.ref.log_term(gid, prev)
                        if prev_t < 0:
                            prev, prev_t = st.epoch_index, st.epoch_term
                    elif mode < 0.9:     # mismatching prev
                        prev, prev_t = last + int(rng.integers(1, 4)), max(term, 1)
                    else:                # below / at the epoch
                        prev, prev_t = st.epoch_index, st.epoch_term
                    if prev == 0:
                        prev_t = 0
                    n_ent = int(rng.integers(0, 5))
                    base_t = max(prev_t, 1)
                    ent = []
                    for _ in range(n_ent):
                        if rng.random() < 0.2:
                            base_t += 1
                        ent.append(min(base_t, max(t, base_t)))
                    first = None if rng.random() < 0.95 else prev + 1 + int(rng.integers(1, 3))
                    peer = st.current_leader if (st.current_leader >= 0 and rng.random() < 0.9) else self._peer()
                    commit, draw = int(rng.integers(0, last + 3)), int(rng.integers(900, 1801))
                    if self.near_commit:
                        commit = max(prev, st.commit_index) + int(self.aux.integers(0, n_ent + 3))
                        draw = draw if self.aux.random() < 0.3 else 0
                    ib.ae_request(r, i, self.now, peer, t, prev, prev_t, ent, leader_commit=commit, first_index=first,
                                  rand=draw)
                elif u < 0.85:
                    t = term + int(rng.choice([-1, 0, 1, 1, 2]))
                    li = st.last_index + int(rng.integers(-1, 2)) if st.last_index >= st.first_index else st.epoch_index + int(rng.integers(0, 2))
                    lt = max(0, st.last_term + int(rng.integers(-1, 2)))
                    fn = ib.prevote_request if rng.random() < 0.5 else ib.vote_request
                    fn(r, i, self.now, self._peer(), max(t, 0), max(li, 0), lt, rand=int(rng.integers(900, 1801)))
                elif u < 0.90:
                    t = term + int(rng.choice([-1, 0, 0, 1]))
                    ib.is_request(r, i, self.now, self._peer(), max(t, 0), st.epoch_index + 5, st.epoch_term, bool(rng.integers(0, 2)),
                                  rand=int(rng.integers(900, 1801)))
                else:
                    has = st.last_index >= st.first_index
                    hi = st.last_index if has else st.epoch_index
                    idx = int(rng.integers(max(st.epoch_index - 1, 0), hi + 2))
                    t = self.ref.log_term(gid, idx)
                    ib.flush(r, i, self.now, idx, t if t >= 0 else max(st.epoch_term, 1))
                # lane events: answer some owed replies (in order per lane), sometimes forge
                owed = self.pending.get(i, [])
                used = set()
                keep = []
                for (f, kind, inc, ep, la) in owed:
                    if f in used or rng.random() < 0.35:
                        keep.append((f, kind, inc, ep, la))
                        continue
                    used.add(f)
                    v = rng.random()
                    outcome = OUT_OK if v < 0.9 else (OUT_ERROR if v < 0.95 else OUT_CANCELED)
                    rt = term if rng.random() < 0.93 else term + int(rng.integers(1, 4))
                    succ = rng.random() < 0.85
                    self.now += 1
                    if kind in (EV_AE_ACK, EV_IS_ACK):
                        ib.ack(r, i, f, self.now, inc, rt, succ, ep, la, outcome=outcome, snapshot=kind == EV_IS_ACK)
                    else:
                        ib.vote_reply(r, i, f, self.now, inc, rt, succ, outcome=outcome, pre=kind == EV_PV_REPLY)
                if len(keep) > 4 * F:
                    keep = keep[-4 * F:]
                self.pending[i] = keep
        return ib

    def _steady(self, ib: abi.Inbox, r: int, i: int, st):
        """A steady position: SUBMIT / keepAlive ops and replies in the group's own term, nearly all successful."""
        aux = self.aux
        u = aux.random()
        if st.role != ROLE_LEADER:
            ib.timeout(r, i, self.now, rand=int(aux.integers(900, 1801)))
        elif u < 0.6:
            ib.submit(r, i, self.now, count=int(aux.integers(1, 4)))
        elif u < 0.8:
            ib.timeout(r, i, self.now)
        used, keep = set(), []
        for (f, kind, inc, ep, la) in self.pending.get(i, []):
            if f in used:
                keep.append((f, kind, inc, ep, la))
                continue
            used.add(f)
            self.now += 1
            if kind in (EV_AE_ACK, EV_IS_ACK):
                ib.ack(r, i, f, self.now, inc, st.current_term, aux.random() < 0.95, ep, la, snapshot=kind == EV_IS_ACK)
            else:
                ib.vote_reply(r, i, f, self.now, inc, st.current_term, True, pre=kind == EV_PV_REPLY)
        self.pending[i] = keep[-4 * self.F:]


# ---------------------------------------------------------------------------------------------
# initial states
# ---------------------------------------------------------------------------------------------
E40, T31, T33 = 1 << 40, 1 << 31, 1 << 33


def wide_init(G, big=(), terms_mod=7) -> np.ndarray:
    """Groups in `big` open with a log that starts near 2^40 and a term of at least 2^31."""
    init = init_array(G, terms=np.arange(G) % terms_mod)
    big = np.asarray(list(big), dtype=np.int64)
    if len(big):
        t = T31 + (big % 5)
        init["term"][big] = t
        init["epoch_index"][big] = E40 + big
        init["epoch_term"][big] = t
        init["first_index"][big] = E40 + big + 1
        init["last_index"][big] = E40 + big + 2
        init["last_term"][big] = t
        init["commit_index"][big] = E40 + big
    return init


# ---------------------------------------------------------------------------------------------
# poisoned-outbox driver: both sides step into outboxes whose every byte starts as POISON, so a cell one side writes
# and the other leaves alone differs even when its right value is 0; cells neither side writes still compare equal
# ---------------------------------------------------------------------------------------------
POISON = 0xA5


def gcols(ib: abi.Inbox, G: int) -> int:
    """Entries of a per-group outbox column: n under RAFTING_INBOX_COMPACT_GROUPS, else max_groups."""
    return ib.n if ib.gids is not None and ib.flags & abi.INBOX_COMPACT_GROUPS else G


def poisoned_outbox(ib: abi.Inbox, F: int, G: int, fill=POISON) -> abi.Outbox:
    out = abi.Outbox(ib.rows, ib.n, F, gcols(ib, G))
    for name, *_ in abi.Outbox.ROW_COLS + abi.Outbox.GROUP_COLS:
        getattr(out, name).view(np.uint8).fill(fill)
    return out


class OracleSUT:
    """The CPU oracle stepping into a poisoned outbox."""

    def __init__(self, cfg: abi.Cfg, fill=POISON, threads=8):
        from oracle import binding
        self.cfg, self.F, self.G, self.fill, self.threads = cfg, cfg.replicas - 1, cfg.max_groups, fill, threads
        self.o = binding.Oracle(cfg)

    def open_bulk(self, first, inits):
        self.o.open_bulk(first, inits)

    def step(self, ib: abi.Inbox) -> abi.Outbox:
        return self.o.step(ib, threads=self.threads, out=poisoned_outbox(ib, self.F, self.G, self.fill))

    def export(self, gid):
        return self.o.export(gid)

    def log_term(self, gid, index):
        return self.o.log_term(gid, index)

    def export_all(self):
        return [self.o.export(g) for g in range(self.G)]


class EngineSUT:
    """The CUDA engine stepped through rafting_step_device: inbox and poisoned outbox live in device memory."""

    def __init__(self, cfg: abi.Cfg, fill=POISON):
        import torch
        from rafting_b200 import engine
        self.cfg, self.F, self.G, self.fill = cfg, cfg.replicas - 1, cfg.max_groups, fill
        self.e = engine.Engine(cfg)
        self.dev = torch.device("cuda", cfg.device)

    def open_bulk(self, first, inits):
        self.e.open_bulk(first, inits)

    def step(self, ib: abi.Inbox) -> abi.Outbox:
        import torch
        from rafting_b200 import devbatch
        din = devbatch.DevInbox.from_host(ib, self.dev)
        dout = devbatch.DevOutbox(ib.rows, ib.n, self.F, gcols(ib, self.G), self.dev, fill=self.fill)
        torch.cuda.synchronize()
        self.e.step_device(din.as_c(), dout.as_c())
        torch.cuda.synchronize()
        return dout.to_host()

    def export(self, gid):
        return self.e.export(gid)

    def export_all(self):
        return self.e.export_bulk(0, self.G)


def assert_all_states_equal(ref, sut, F, where=""):
    for gid, (sa, sb) in enumerate(zip(ref.export_all(), sut.export_all())):
        if state_bytes(sa, F) != state_bytes(sb, F):
            da, db = sa.as_dict(), sb.as_dict()
            raise AssertionError(f"group {gid} state differs {where}: { {k: (da[k], db[k]) for k in da if da[k] != db[k]} }")


# ---------------------------------------------------------------------------------------------
# the fuzz matrix: every kernel and launch mode of launch_step (tests/launch_model.py) under every event kind
# ---------------------------------------------------------------------------------------------
@dataclass(frozen=True)
class FuzzCase:
    id: str
    R: int
    G: int
    seed: int
    steps: int = 30
    cpu_steps: int = 10        # the oracle-on-both-sides rehearsal (tests/test_fuzz_matrix_cpu.py)
    rows: int = 3
    local_slot: int = 0
    pre_vote: bool = True
    n_active: int = 0          # > 0: an active list of that many positions ...
    tail: int = 0              # ... of which the last `tail` hold ids >= G
    compact: bool = False      # RAFTING_INBOX_COMPACT_GROUPS on the active list
    leader_share: float = 0.0  # > 0: elect every group first, then keep this share steady
    sweep_every: int = 0
    stray: int = 0
    wide: bool = False         # a third of the groups near 2^40 / terms >= 2^31, fuzz times 2^33 ms later
    state_every: int = 10
    legacy: bool = False       # a stream the suite has replayed unchanged since before the knobs existed

    @property
    def n(self):
        return self.n_active or self.G

    def cfg(self) -> abi.Cfg:
        return abi.make_cfg(replicas=self.R, local_slot=self.local_slot, max_groups=self.G, max_rows=self.rows,
                            pre_vote=self.pre_vote, entry_pool_cap=self.rows * self.n * 8)

    def init(self) -> np.ndarray:
        return wide_init(self.G, range(0, self.G, 3) if self.wide else (), terms_mod=3)

    def gids(self):
        if not self.n_active:
            return None
        pick = np.random.default_rng([self.seed, 0x61D5]).choice(self.G, self.n_active - self.tail, replace=False)
        return np.concatenate([np.sort(pick), self.G + 3 * np.arange(self.tail)]).astype(np.uint32)


def _u(id, R, G, seed, **kw):
    return FuzzCase(id, R, G, seed, sweep_every=kw.pop("sweep_every", 7), stray=kw.pop("stray", 4), **kw)


def _s(id, R, G, seed, **kw):
    return FuzzCase(id, R, G, seed, steps=kw.pop("steps", 14), cpu_steps=kw.pop("cpu_steps", 8), leader_share=0.35,
                    sweep_every=kw.pop("sweep_every", 11), stray=kw.pop("stray", 3), state_every=5, **kw)


# steps launched without a class sort (n < 2048, a NO_REQUESTS step, or R > 9)
FUZZ_UNSORTED = [
    FuzzCase("3-0-True-1", 3, 48, 1, steps=60, legacy=True),
    FuzzCase("3-2-False-2", 3, 48, 2, steps=60, local_slot=2, pre_vote=False, legacy=True),
    FuzzCase("5-2-True-3", 5, 48, 3, steps=60, local_slot=2, legacy=True),
    FuzzCase("4-1-True-4", 4, 48, 4, steps=60, local_slot=1, legacy=True),
    FuzzCase("7-6-False-5", 7, 48, 5, steps=60, local_slot=6, pre_vote=False, legacy=True),
    _u("R2-G777", 2, 777, 21, local_slot=1),
    _u("R2-G777-wide", 2, 777, 22, wide=True),
    _u("R3-G777", 3, 777, 23, local_slot=1),
    _u("R3-G777-wide", 3, 777, 24, wide=True, pre_vote=False),
    _u("R3-n2047", 3, 2047, 25, steps=16),
    _u("R4-G777-wide", 4, 777, 26, local_slot=3, wide=True),
    _u("R6-G777", 6, 777, 27, local_slot=2),
    _u("R6-G777-wide", 6, 777, 28, wide=True),
    _u("R9-G777", 9, 777, 29, local_slot=8),
    _u("R9-n2047", 9, 2047, 30, steps=16),
    _u("R10-G300", 10, 300, 31, local_slot=4),
    _u("R17-G300-wide", 17, 300, 32, wide=True),
    _u("R33-G300", 33, 300, 33, local_slot=32, pre_vote=False),
    _u("R33-G300-wide", 33, 300, 34, wide=True),
    _u("R3-active1500-compact", 3, 4096, 35, n_active=1500, tail=37, compact=True, steps=16),
]

# steps that may carry requests over >= 2048 positions at R <= 9: classify_kernel sorts them
FUZZ_SORTED = [
    FuzzCase("3-11", 3, 2304, 11, steps=14, cpu_steps=6, local_slot=1, legacy=True),
    FuzzCase("5-12", 5, 2304, 12, steps=14, cpu_steps=6, local_slot=1, legacy=True),
    _s("R2-G2304", 2, 2304, 41),
    _s("R2-G2304-wide", 2, 2304, 42, local_slot=1, wide=True),
    _s("R3-n2048", 3, 2048, 43, local_slot=2),
    _s("R3-G2304-wide", 3, 2304, 44, wide=True),
    _s("R4-G2304-wide", 4, 2304, 45, local_slot=1, wide=True),
    _s("R6-G2304", 6, 2304, 46, local_slot=5),
    _s("R9-G2304-wide", 9, 2304, 47, local_slot=3, wide=True),
    _s("R9-n2048", 9, 2048, 48),
    _s("R3-active2100", 3, 4096, 49, n_active=2100, tail=40),
    _s("R5-active2100-compact", 5, 4096, 50, n_active=2100, tail=40, compact=True),
    _s("R9-active2100-compact", 9, 4096, 51, n_active=2100, tail=40, compact=True),
]


@dataclass
class Coverage:
    roles: set = field(default_factory=set)
    errs: set = field(default_factory=set)
    classes: list = field(default_factory=list)     # per class-sorted step: positions per class
    launches: set = field(default_factory=set)      # (kernels, mode) of launch_model.kernels


def run_fuzz_case(case: FuzzCase, sut_factory, steps=None, ref_factory=OracleSUT) -> Coverage:
    """Drives `case` through a poisoned reference (the oracle) and a poisoned SUT, comparing every outbox, the state of a
    spread of groups every `state_every` steps and of every group at the end."""
    from tests import launch_model
    cfg, F, G = case.cfg(), case.R - 1, case.G
    ref, sut = ref_factory(cfg), sut_factory(cfg)
    init = case.init()
    ref.open_bulk(0, init)
    sut.open_bulk(0, init)
    out = None
    if case.leader_share:
        w1 = workload.make_wl(case.seed, 1, G, F, local_slot=case.local_slot)
        out = elect_all(ref, w1)
        assert_outbox_equal(out, elect_all(sut, w1), where=f"{case.id}: election")
    gids = case.gids()
    fz = Fuzzer(cfg, ref, seed=case.seed, rows=case.rows, gids=gids, leader_share=case.leader_share,
                sweep_every=case.sweep_every, stray_requests=case.stray, t0=T33 if case.wide else 0)
    # the cells a step writes for certain: the group columns of the groups that take part, the rows of their positions
    pos = np.arange(fz.n) if gids is None else np.flatnonzero(gids < G)
    grp = pos if gids is None or case.compact else gids[pos]
    spread = np.arange(0, G, max(1, G // 97))
    if gids is not None:
        spread = np.union1d(spread, gids[pos][:64])
    cov = Coverage()
    for k in range(case.steps if steps is None else steps):
        ib = fz.make(out)
        if case.compact:
            ib.flags |= abi.INBOX_COMPACT_GROUPS
        launch = launch_model.kernels(case.R, ib.n, ib.flags)
        cov.launches.add(launch)
        if launch[1] == "class-sorted":
            cov.classes.append(np.bincount(launch_model.classes(ref, ib), minlength=launch_model.NCLS))
        out = ref.step(ib)
        assert_outbox_equal(out, sut.step(ib), where=f"{case.id}: fuzz step {k}")
        cov.roles |= set((out.role_word[grp] & 3).tolist())
        cov.errs |= set(((out.rep_meta[:, pos] >> 8) & 0xFF).ravel().tolist())
        if k % case.state_every == case.state_every - 1:
            assert_states_equal(ref, sut, spread.tolist(), F, where=f"{case.id}: fuzz step {k}")
    assert_all_states_equal(ref, sut, F, where=f"{case.id}: end of the fuzz")
    return cov


def check_coverage(case: FuzzCase, cov: Coverage):
    """The steering reached what the case is there for: every role, several error paths and, in a class-sorted case
    whose leaders are steered, every class most of the time and the two leader classes each wider than a 128-thread
    block in some step."""
    assert cov.roles == {0, 1, 2}, cov.roles
    assert len(cov.errs) > 3, cov.errs
    if case.leader_share:
        c = np.array(cov.classes)
        assert len(c), "no class-sorted step"
        assert ((c > 0).all(axis=1)).mean() > 0.5, c.tolist()
        assert c[:, 2].max() > 128 and c[:, 3].max() > 128, c.tolist()
