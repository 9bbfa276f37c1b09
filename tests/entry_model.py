"""A plain restatement of the HBM entry buffer (rafting_b200/csrc/seglog.cuh), for the entry-buffer suites.
TEST INFRASTRUCTURE ONLY (same rule as raft_oracle.c).  It never reads the engine's state: it is driven by the calls a test
makes (appends with their refs and blob, trims with the stored key ranges the CPU oracle exports) and predicts, exactly,
what every read path of the entry buffer returns and what rafting_log_stats counts.

  arena      a record is 32 + align16(len) bytes; one that would straddle a segment starts at the next boundary; an append
             is cut into sub-batches that each end within nseg segments of the start of the head's segment; the newest nseg
             segments are resident
  host index per group a window [base, base + size) of at most WINDOW indices; the latest put wins in batch order; an
             index one WINDOW or more past the window's end, or so far below it that the newest WINDOW indices would not hold
             it, starts a new window; a window grown past WINDOW keeps its newest WINDOW indices; rafting_log_trim drops what
             lies below each group's lowest stored key
  ring       slot (gid, index & (K - 1)) names the newest record ever published there
  hit rule   the device serves (gid, i) iff the host index holds it, its record is resident and that record is the one its
             ring slot names; every other entry is served by the host (host_served)

Visible reads (rafting_log_read) follow oracle/payload_model.PayloadLog, bounded by the stored key range and the blob cap.
"""
from __future__ import annotations

import re
from dataclasses import dataclass, field

import numpy as np

from rafting_b200 import abi

WINDOW = 1 << 22                       # SEGLOG_INDEX_WINDOW: indices one group's host index spans at most
HDR = 32                               # SegHdr
ABSENT = 0xFFFFFFFF
ENTRY_REF = np.dtype([("gid", "<u4"), ("len", "<u4"), ("index", "<i8"), ("term", "<i8"), ("blob_off", "<u8")])


def a16(n: int) -> int:
    return (n + 15) & ~15


def window_constant(seglog_source: str) -> int:
    """SEGLOG_INDEX_WINDOW as seglog.cuh states it"""
    m = re.search(r"SEGLOG_INDEX_WINDOW\s*=\s*(?:\(int64_t\))?\s*1\s*<<\s*(\d+)\s*;", seglog_source)
    return 1 << int(m.group(1))


def plan_ranges(d: abi.Outbox, F: int, n: int, gids):
    """(lane slots, gids, first indices, counts) of the AE plans with entries in the dense plan columns of an outbox"""
    m = d.plan_meta.reshape(-1)
    c = np.where((m & 0xF) == abi.PLAN_AE, (m >> 16) & 0xFFFF, 0).astype(np.int64)
    t = np.flatnonzero(c)
    pos = (t // F) % n
    g = pos if gids is None else np.asarray(gids, np.int64)[pos]
    return t, g, d.plan_pp.reshape(-1)["x"][t] + 1, c[t]


def dense_ranges(e, slot: int, rows: int, n: int, gids):
    """plan_ranges of the step last waited for in the engine's slot (rafting_step_fetch_dense)"""
    d = abi.Outbox(rows, n, e.F, n)
    e.step_fetch_dense(slot, d.as_c())
    return plan_ranges(d, e.F, n, gids)


@dataclass
class Rec:
    off: int                           # logical offset of the record
    len: int
    term: int
    payload: bytes


@dataclass
class Group:
    base: int = 0
    size: int = 0                      # the window [base, base + size); entries holds the indices stored in it
    entries: dict = field(default_factory=dict)
    trimmed_to: int = 0                # the highest base a trim or a cut gave the window (coverage only)


class EntryModel:
    def __init__(self, segment_bytes: int, hbm_segments: int, ring_slots: int, entry_file: bool = False, cold_max: int = 0):
        self.S, self.nseg, self.K = segment_bytes, hbm_segments, ring_slots
        self.file, self.cold_max = entry_file, cold_max
        self.head = self.appended = self.spilled_upto = 0
        self.stats = dict(appended=0, head=0, spilled_bytes=0, indexed=0, trimmed=0, cold_freed_bytes=0, spills_skipped=0)
        self.groups: dict[int, Group] = {}
        self.ring: dict[tuple[int, int], int] = {}
        self.live: dict[int, int] = {}                 # live records per logical segment
        self.cold: set[int] = set()                    # segments with a pinned host copy
        self.lru: list[int] = []
        self.seen: set[str] = set()                    # the cases the calls so far reached (coverage)

    # ---- arena ----------------------------------------------------------------------------------------------------
    def resident(self, off: int) -> bool:
        newest = (self.head - 1) // self.S if self.head else 0
        return off // self.S + self.nseg > newest

    def tier(self, rec: Rec) -> str:
        if self.resident(rec.off):
            return "hbm"
        return "cold" if rec.off // self.S in self.cold else "file"

    def _spill_for(self, new_head: int):
        last = (new_head - 1) // self.S
        while last >= self.nseg and self.spilled_upto <= last - self.nseg:
            s = self.spilled_upto
            self.spilled_upto += 1
            if self.live.get(s, 0) == 0:
                self.stats["spills_skipped"] += 1
                self.seen.add("spill skipped")
                continue
            self.cold.add(s)
            self.stats["spilled_bytes"] += self.S
            self.lru.append(s)
            while self.cold_max and self.file and len(self.lru) > self.cold_max:
                v = self.lru[0]
                if v in self.cold:
                    if (v + 1) * self.S > self.head:
                        break
                    self.cold.discard(v)
                self.lru.pop(0)

    # ---- host index -----------------------------------------------------------------------------------------------
    def _drop(self, rec: Rec):
        self.live[rec.off // self.S] -= 1
        self.stats["indexed"] -= 1

    def _put(self, gid: int, index: int, rec: Rec):
        g = self.groups.setdefault(gid, Group())
        if g.size == 0:
            if index < g.trimmed_to:
                self.seen.add("restart below a trimmed empty window")
            g.base = index
        if index < g.base + g.size - WINDOW or index >= g.base + g.size + WINDOW:
            if index < g.base and g.size == WINDOW and index >= g.base - WINDOW:
                self.seen.add("restart below a full window")
            elif index < g.base:
                self.seen.add("backward restart after a trim above the window" if g.base > WINDOW + 1 and g.trimmed_to == g.base
                              else "backward restart")
            else:
                self.seen.add("forward restart")
            for r in g.entries.values():
                self._drop(r)
            g.entries.clear()
            g.base, g.size = index, 0
        if index < g.base:
            g.size += g.base - index
            g.base = index
        if index >= g.base + g.size:
            g.size = index - g.base + 1
        if g.size > WINDOW:
            cut = g.size - WINDOW
            for i in [i for i in g.entries if i < g.base + cut]:
                self._drop(g.entries.pop(i))
            g.base += cut
            g.size = WINDOW
            g.trimmed_to = g.base
            self.seen.add("cut")
        assert g.base <= index < g.base + g.size <= g.base + WINDOW, (gid, index, g.base, g.size)
        old = g.entries.get(index)
        if old is None:
            self.stats["indexed"] += 1
        else:
            self.live[old.off // self.S] -= 1
        self.live[rec.off // self.S] = self.live.get(rec.off // self.S, 0) + 1
        g.entries[index] = rec

    def find(self, gid: int, index: int) -> Rec | None:
        g = self.groups.get(gid)
        return None if g is None else g.entries.get(index)

    # ---- calls ----------------------------------------------------------------------------------------------------
    def append(self, refs: np.ndarray, blob: bytes):
        """rafting_log_append(refs, blob) of valid refs (ENTRY_REF records)"""
        n, done = len(refs), 0
        offs = refs["blob_off"].astype(np.int64)
        if len(set(offs.tolist())) < n:
            self.seen.add("shared source")
        if (offs % 16 != 0).any():
            self.seen.add("unaligned source")
        keys = list(zip(refs["gid"].tolist(), refs["index"].tolist()))
        if len(set(keys)) < n:
            self.seen.add("duplicate in a batch")
        while done < n:
            head, m, sub = self.head, 0, []
            end = (self.head // self.S + self.nseg) * self.S    # the arena, from the start of the head's segment
            for i in range(done, n):
                r = refs[i]
                ln = int(r["len"])
                rec = HDR + a16(ln)
                h2 = head
                if h2 // self.S != (h2 + rec - 1) // self.S:
                    h2 = (h2 // self.S + 1) * self.S
                    self.seen.add("tail skip")
                if h2 + rec > end:
                    break
                if rec == self.S:
                    self.seen.add("record fills a segment")
                if ln == 0:
                    self.seen.add("zero length")
                if int(r["index"]) >= 1 << 32:
                    self.seen.add("index >= 2^32")
                o = int(r["blob_off"])
                self._put(int(r["gid"]), int(r["index"]), Rec(h2, ln, int(r["term"]), bytes(blob[o:o + ln])))
                sub.append((int(r["gid"]), int(r["index"]), h2))
                head = h2 + rec
                m += 1
            assert m, "arena too small for a single record"
            if m < n - done:
                self.seen.add("sub-batch split")
            self._spill_for(head)
            for gid, index, off in sub:
                k = (gid, index & (self.K - 1))
                self.ring[k] = max(self.ring.get(k, 0), off + 1)
            self.head = head
            self.appended += m
            done += m
        self.stats["appended"], self.stats["head"] = self.appended, self.head

    def trim(self, ranges: dict, first_gid: int, count: int):
        """rafting_log_trim(first_gid, count); ranges[gid] = (first_index, last_index, empty) as the oracle exports them"""
        dropped = freed = 0
        for gid in range(first_gid, first_gid + count):
            g = self.groups.get(gid)
            if g is None or g.size == 0:
                continue
            lo, hi, empty = ranges[gid]
            cut = min((hi + 1 if empty else lo) - g.base, g.size)
            if cut <= 0:
                continue
            for i in [i for i in g.entries if i < g.base + cut]:
                self._drop(g.entries.pop(i))
                dropped += 1
            g.base += cut
            g.size -= cut
            g.trimmed_to = g.base
            if g.base > WINDOW + 1:
                self.seen.add("trim above the window")
        for s in sorted(self.cold):
            if self.live.get(s, 0) == 0:
                self.cold.discard(s)
                freed += self.S
        self.stats["trimmed"] += dropped
        self.stats["cold_freed_bytes"] += freed
        return dropped, freed

    def served(self, gid: int, index: int) -> bool:
        """the hit rule: the device serves (gid, index)"""
        r = self.find(gid, index)
        if r is None or not self.resident(r.off):
            return False
        if self.ring[(gid, index & (self.K - 1))] != r.off + 1:
            self.seen.add("ring slot holds a newer index")
            return False
        return True

    def read(self, gid: int, first: int, max_n: int, blob_cap: int, stored):
        """rafting_log_read -> ([(index, term, payload)], tiers of the non-empty payloads read); stored = (lo, hi, empty)"""
        lo, hi, empty = stored
        if empty:
            lo, hi = 1, 0
        out, tiers, used = [], [], 0
        i = first
        while len(out) < max_n and lo <= i <= hi:
            r = self.find(gid, i)
            if r is None or used + r.len > blob_cap:
                break
            out.append((i, r.term, r.payload))
            if r.len:
                tiers.append(self.tier(r))
            used += a16(r.len)
            i += 1
        for t in tiers:
            self.seen.add(f"{t} read")
        return out, tiers

    def refs(self, ranges):
        """rafting_log_gather's refs for ranges [(gid, first, count)] -> (ENTRY_REF array, payloads, aligned total)"""
        n = sum(c for _, _, c in ranges)
        out = np.zeros(n, ENTRY_REF)
        pays, used, k = [], 0, 0
        for gid, first, count in ranges:
            for i in range(first, first + count):
                r = self.find(gid, i)
                out[k] = (gid, ABSENT, i, 0, used) if r is None else (gid, r.len, i, r.term, used)
                pays.append(None if r is None else r.payload)
                if r is not None:
                    used += a16(r.len)
                k += 1
        return out, pays, used

    def gather(self, ranges, blob_cap: int):
        """rafting_log_gather and rafting_log_gather_begin/_wait -> (refs, payloads, bytes, host_served, fits)"""
        refs, pays, need = self.refs(ranges)
        host = sum(1 for r in refs if not self.served(int(r["gid"]), int(r["index"])))
        return refs, pays, need, host, need <= blob_cap

    def gather_step(self, t, g, f, c):
        """rafting_log_gather_step_begin/_wait over plan_ranges -> (refs, payloads, bytes, host_served, plan records): the
        device-served payloads first in ref order, then the host-served ones, each miss at the running total in its turn"""
        refs, pays, _ = self.refs(list(zip(g.tolist(), f.tolist(), c.tolist())))
        hit = [self.served(int(r["gid"]), int(r["index"])) for r in refs]
        off = 0
        for k, r in enumerate(refs):
            if hit[k]:
                r["blob_off"] = off
                off += a16(int(r["len"]))
        for k, r in enumerate(refs):
            if not hit[k]:
                r["blob_off"] = off
                if r["len"] != ABSENT:
                    off += a16(int(r["len"]))
        plans = np.zeros(len(t), abi.PLAN_REF)
        if len(t):
            plans["slot"], plans["count"] = t, c
            plans["first"] = np.concatenate([[0], np.cumsum(c)[:-1]])
        return refs, pays, off, hit.count(False), plans

    def export_kv(self, gid: int, index: int):
        """rafting_log_export_kv -> (key, value) or None (RAFTING_E_INVAL)"""
        r = self.find(gid, index)
        if r is None:
            return None
        if r.len:
            self.seen.add(f"{self.tier(r)} read")
        return index.to_bytes(8, "big"), (r.term & (1 << 64) - 1).to_bytes(8, "big") + r.payload


# ---- op streams: the entry-buffer fuzz cases, driven through the oracle and this model (and, on a GPU, the engine) ----------
@dataclass(frozen=True)
class Case:
    name: str
    segment_bytes: int
    hbm_segments: int
    ring_slots: int
    entry_file: bool = False
    cold_max: int = 0
    wide: bool = False
    seed: int = 1
    ops: int = 60
    G: int = 32

    @property
    def log(self) -> dict:
        return dict(segment_bytes=self.segment_bytes, hbm_segments=self.hbm_segments, ring_slots=self.ring_slots)


CASES = [
    Case("4096x2 K1", 4096, 2, 1, seed=11),
    Case("4096x3 K2", 4096, 3, 2, seed=12),
    Case("8192x4 K16 file", 8192, 4, 16, entry_file=True, cold_max=1, seed=13),
    Case("65536x8 K64 wide", 65536, 8, 64, wide=True, seed=14),
]

L0 = 3000                              # stored keys 1..L0 (or base + 1 .. base + L0) of every group at open
HIGH = 5_000_000                       # groups 1 and 2 start their log here: a trim leaves their window above WINDOW + 1
WIDE = (1 << 32) + 5                   # upper half of a wide case's groups start here


def stream_init(case: Case):
    from tests import harness
    init = harness.init_array(case.G, terms=1)
    init["last_index"], init["last_term"] = L0, 1
    bases = np.zeros(case.G, np.int64)
    bases[1:3] = HIGH
    if case.wide:
        bases[case.G // 2:] = WIDE
    init["epoch_index"] = bases
    init["epoch_term"] = np.where(bases > 0, 1, 0)
    init["commit_index"] = bases
    init["first_index"] = bases + 1
    init["last_index"] = bases + L0
    return init, bases


def payload_len(rng, S: int) -> int:
    r = rng.random()
    if r < 0.1:
        return 0
    if r < 0.7:
        return int(rng.integers(1, 65))
    if r < 0.9:
        return int(rng.integers(65, 700))
    if r < 0.95:
        return S - HDR                                 # fills a segment exactly
    return int(rng.integers(S // 3, S // 2))           # leaves a tail the next record skips


def adversarial_batch(rng, entries, S: int):
    """entries [(gid, index, term, len)] -> (refs, blob): payloads at odd, shared and overlapping offsets of one random blob,
    refs out of blob order; a share of them 16-byte aligned"""
    lens = [x[3] for x in entries]
    size = max(sum(lens) // 2 + max(lens + [0]) + 64, 64)
    blob = rng.bytes(size)
    refs = np.zeros(len(entries), ENTRY_REF)
    offs = []
    for k, (gid, index, term, ln) in enumerate(entries):
        r = rng.random()
        if offs and r < 0.15:
            o = offs[int(rng.integers(0, len(offs)))]
            o = o if o + ln <= size else 0
        elif r < 0.35:
            o = int(rng.integers(0, (size - ln) // 16 + 1)) * 16
        else:
            o = int(rng.integers(0, size - ln + 1))
        offs.append(o)
        refs[k] = (gid, ln, index, term, o)
    return refs, blob


class Stream:
    """One case's op stream.  Each op changes the oracle (steps, opens, closes) and the model, and hands the same call to
    `eng` (an object with the Engine's methods plus append_raw(refs, blob)) when one is given.  ops() yields a label per op."""

    def __init__(self, case: Case, eng=None):
        from oracle import binding
        self.case, self.eng = case, eng
        self.rng = np.random.default_rng(case.seed)
        self.cfg = abi.make_cfg(replicas=3, max_groups=case.G, max_rows=1, entry_pool_cap=64)
        self.o = binding.Oracle(self.cfg)
        init, self.bases = stream_init(case)
        self.o.open_bulk(0, init)
        self.m = EntryModel(case.segment_bytes, case.hbm_segments, case.ring_slots, case.entry_file, case.cold_max)
        if eng is not None:
            eng.open_bulk(0, init)
            eng.log_config(**case.log)
            if case.entry_file:
                eng.log_store_open(eng.entry_path, cold_max_segments=case.cold_max)
        self.next = self.bases + 1                      # per group: one past the highest index appended in its window
        self.spots: list[tuple[int, int]] = []          # (gid, index) places worth gathering around
        self.now = 0
        self.crng = np.random.default_rng(case.seed + 1000)   # the checks' choices: the op stream does not depend on them

    # ---- what the oracle stores -----------------------------------------------------------------------------------
    def stored(self, gid: int):
        s = self.o.export(gid)
        return int(s.first_index), int(s.last_index), int(s.term_runs) == 0

    def _step(self, ib: abi.Inbox):
        self.o.step(ib)
        if self.eng is not None:
            self.eng.step(ib)

    # ---- ops ------------------------------------------------------------------------------------------------------
    def append(self, entries):
        refs, blob = adversarial_batch(self.rng, entries, self.case.segment_bytes)
        self.m.append(refs, blob)
        if self.eng is not None:
            self.eng.append_raw(refs, blob)
        for gid, index, _, _ in entries:
            self.next[gid] = max(self.next[gid], index + 1)
            if self.rng.random() < 0.05:
                self.spots.append((gid, index))

    def op_append(self):
        n = int(self.rng.integers(1, 301))
        ents = []
        while len(ents) < n:
            gid = int(self.rng.integers(0, self.case.G))
            lo = int(self.next[gid]) - int(self.rng.integers(0, 6))
            g = self.m.groups.get(gid)
            # Kept out on purpose: a window that grows back below the base a trim or cut gave it, without restarting.  The
            # engine's index floor stays at that base, so the device leaves those entries to the host (the bytes are right),
            # where the hit rule above says the device serves them: a known difference from the intended rule.
            if g is not None and g.trimmed_to and (g.size == 0 or g.trimmed_to == g.base) and lo > g.trimmed_to - WINDOW:
                lo = max(lo, g.trimmed_to)
            run = int(self.rng.integers(1, 24))
            for i in range(max(lo, 1), max(lo, 1) + run):
                ents.append((gid, i, 1, payload_len(self.rng, self.case.segment_bytes)))
        ents = ents[:n]
        for _ in range(int(self.rng.integers(0, 6))):        # duplicates inside the batch: the later one wins
            gid, i, t, _ = ents[int(self.rng.integers(0, len(ents)))]
            ents.append((gid, i, t, payload_len(self.rng, self.case.segment_bytes)))
        order = self.rng.permutation(len(ents))
        self.append([ents[k] for k in order])
        return f"append {len(ents)}"

    def op_far(self, kind: str, gid: int):
        g = self.m.groups.get(gid)
        if kind == "forward":
            index = int(self.next[gid]) + WINDOW + int(self.rng.integers(0, 1000))
            if self.case.wide and self.rng.random() < 0.5 and g is not None and g.entries:
                index = min(g.entries) + (1 << 32)          # same low 32 bits, same ring slot as an entry it drops
        elif kind == "backward":
            index = 1 + int(self.rng.integers(0, 50))
        elif kind == "under":                               # one past a full window's end cuts its base; the old base is then
            top, low = g.base + g.size, g.base              # below the newest WINDOW indices: a new window
            self.spots.append((gid, low))
            self.append([(gid, top, 1, payload_len(self.rng, self.case.segment_bytes)),
                         (gid, low, 1, payload_len(self.rng, self.case.segment_bytes)),
                         (gid, low + 1, 1, payload_len(self.rng, self.case.segment_bytes))])
            self.next[gid] = low + 2
            return f"put under the full window of {gid}"
        else:                                               # cut: past the window by a few indices, not far enough to restart
            index = g.base + WINDOW + 4
        run = int(self.rng.integers(2, 12))
        self.spots += [(gid, index), (gid, index - (1 << 32) if index > 1 << 32 else index)]
        self.append([(gid, index + j, 1, payload_len(self.rng, self.case.segment_bytes)) for j in range(run)])
        if kind != "cut":
            self.next[gid] = index + run
        return f"{kind} restart of {gid} at {index}" if kind != "cut" else f"cut of {gid}"

    def op_flush(self, gids, trim_all: bool):
        ib = abi.Inbox(1, self.case.G, 2)
        self.now += 1
        for gid in gids:
            lo, hi, empty = self.stored(gid)
            if empty:
                continue
            idx = hi if self.rng.random() < 0.2 else int(self.rng.integers(lo, hi + 1))
            ib.flush(0, gid, 10_000 + self.now, idx, self.o.log_term(gid, idx))
        self._step(ib)
        first, count = (0, self.case.G) if trim_all else (min(gids), max(gids) - min(gids) + 1)
        ranges = {g: self.stored(g) for g in range(first, first + count)}
        want = self.m.trim(ranges, first, count)
        if self.eng is not None:
            got = self.eng.log_trim(first, count)
            assert got == want, f"log_trim({first}, {count}) = {got}, model {want}"
        return f"flush {list(gids)}, trim {first}+{count}"

    def op_conflict(self, gid: int):
        lo, hi, empty = self.stored(gid)
        if empty or hi - lo < 4:
            return "conflict skipped"
        st = self.o.export(gid)
        prev = int(self.rng.integers(lo, hi - 2))
        term = int(st.current_term) + 1
        ib = abi.Inbox(1, self.case.G, 2, ent_cap=8)
        self.now += 1
        ib.ae_request(0, gid, 10_000 + self.now, 1, term, prev, self.o.log_term(gid, prev), [term, term], leader_commit=0)
        self._step(ib)
        assert self.stored(gid)[1] == prev + 2, "the conflicting AppendEntries truncates the suffix"
        self.append([(gid, prev + 1, term, payload_len(self.rng, self.case.segment_bytes)),
                     (gid, prev + 2, term, payload_len(self.rng, self.case.segment_bytes))])
        self.spots.append((gid, prev - 2))
        return f"conflict on {gid} after {prev}"

    def op_reopen(self, gid: int, base: int = 0):
        init = {"term": 1, "first_index": base + 1, "last_index": base + L0, "last_term": 1, "epoch_index": base,
                "epoch_term": 1 if base else 0, "commit_index": base, "now_ms": 0, "rand_ms": 0}
        for sut in (self.o, self.eng) if self.eng is not None else (self.o,):
            sut.close_group(gid)
            sut.open_group(gid, **init)
        self.next[gid] = base + 1
        return f"reopen {gid} at {base + 1}"

    def ops(self):
        """the case's op stream; the fixed ops at fixed places make sure every case reaches the window events"""
        G, rng = self.case.G, self.rng
        fixed = {
            5: lambda: self.op_flush([1, 2], False),
            6: lambda: self.op_flush([1], False),           # group 1 trimmed above the window
            8: lambda: self.op_far("forward", 3),
            12: lambda: self.op_reopen(1),
            13: lambda: self.op_far("backward", 1),         # restart below a base above WINDOW + 1 (the reopened context)
            16: lambda: self.op_far("cut", 4),
            17: lambda: self.op_far("under", 4),
            18: lambda: self.op_flush([2], False),
            19: lambda: self.op_reopen(2),
            20: lambda: self.op_far("backward", 2),
            24: lambda: self.op_conflict(5),
        }
        for k in range(self.case.ops):
            if k in fixed:
                yield fixed[k]()
                continue
            r = rng.random()
            if r < 0.6:
                yield self.op_append()
            elif r < 0.7:
                yield self.op_far("forward", int(rng.integers(0, G)))
            elif r < 0.82:
                gids = sorted(set(int(x) for x in rng.integers(0, G, int(rng.integers(1, 5)))))
                yield self.op_flush(gids, rng.random() < 0.5)
            elif r < 0.9:
                yield self.op_conflict(int(rng.integers(5, G)))
            else:
                yield self.op_reopen(int(rng.integers(5, G)), int(self.bases[int(rng.integers(0, G))]))

    # ---- the reads a check makes ------------------------------------------------------------------------------------
    def random_ranges(self, n: int):
        rng, out = self.crng, []
        for _ in range(n):
            if self.spots and rng.random() < 0.5:
                gid, i = self.spots[int(rng.integers(0, len(self.spots)))]
            else:
                gid = int(rng.integers(0, self.case.G))
                i = int(self.next[gid]) - int(rng.integers(0, 400))
            first = max(1, i - int(rng.integers(0, 8)))
            out.append((gid, first, int(rng.integers(0, 16))))
        return out

    def reads(self, n: int = 3):
        """[(gid, first, max_n, blob_cap)] for rafting_log_read, and [(gid, index)] for rafting_log_export_kv"""
        rng, rd, kv = self.crng, [], []
        for _ in range(n):
            gid = int(rng.integers(0, self.case.G))
            lo, hi, _ = self.stored(gid)
            first = max(lo, int(self.next[gid]) - int(rng.integers(1, 400)))
            rd.append((gid, first, int(rng.integers(1, 80)), int(rng.choice([64, 4096, 1 << 20]))))
            g = self.m.groups.get(gid)
            if g is not None and g.entries:
                keys = sorted(g.entries)
                kv.append((gid, keys[int(rng.integers(0, len(keys)))]))
            kv.append((gid, first))
        return rd, kv
