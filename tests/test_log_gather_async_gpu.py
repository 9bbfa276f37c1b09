"""rafting_log_gather_begin / _wait: the payloads of (gid, first, count) ranges gathered on the device under a ticket.

Every gather is held to rafting_log_gather with the same arguments: the refs must be equal record for record (gid, len, index,
term and blob_off), and the payload bytes at every ref's blob_off equal.  The entries live in every place the entry buffer
keeps them (HBM, a ring slot that caches a newer index, the pinned cold tier, the entry file, trimmed, never appended), the
ranges take every shape an apply loop hands over, and the apply loop of a compact pump runs pipelined: each step's apply
ranges are gathered under a ticket that stays outstanding while the next step runs."""
import ctypes as C

import numpy as np
import pytest

from rafting_b200 import abi, compact, engine, ingest, workload
from tests import edit_pump
from tests import harness
from tests import timers_model as tm

pytestmark = pytest.mark.gpu

ABSENT = 0xFFFFFFFF
_PINNED = []                                       # the pinned tensors behind the views pinned() hands out


def pinned(nbytes: int, dtype, skew: int = 0) -> np.ndarray:
    import torch
    t = torch.zeros(max(nbytes + skew, 16), dtype=torch.uint8, pin_memory=True)
    _PINNED.append(t)
    return t.numpy()[skew:skew + nbytes].view(dtype)


def outputs(kind: str, n_refs: int, blob_cap: int, fill: int = 0):
    """refs and blob in pinned memory (written by the device), pageable memory (staged), or a pinned blob 8 bytes off a
    16-byte boundary (staged)"""
    if kind == "pinned":
        refs, blob = pinned(n_refs * 32, engine.Engine.ENTRY_REF), pinned(blob_cap, np.uint8)
    elif kind == "misaligned":
        refs, blob = pinned(n_refs * 32, engine.Engine.ENTRY_REF), pinned(blob_cap, np.uint8, skew=8)
    else:
        refs, blob = np.zeros(n_refs, engine.Engine.ENTRY_REF), np.zeros(blob_cap, np.uint8)
    blob[:] = fill
    return refs, blob


def arrays(ranges):
    return (np.array([r[0] for r in ranges], np.uint32), np.array([r[1] for r in ranges], np.int64),
            np.array([r[2] for r in ranges], np.uint32))


def reference(e: engine.Engine, g, f, c, blob_cap: int):
    """rafting_log_gather with the same arguments: (refs, blob, bytes)"""
    cap = int(c.sum()) + 1
    refs, blob = np.zeros(cap, e.ENTRY_REF), np.zeros(max(blob_cap, 16), np.uint8)
    if len(g) == 0:
        return refs[:0], blob, 0
    n, nb = C.c_uint32(), C.c_size_t()
    engine._check(engine.lib().rafting_log_gather(e._h, len(g), g.ctypes.data, f.ctypes.data, c.ctypes.data, refs.ctypes.data, cap,
                                                  blob.ctypes.data, blob_cap, C.byref(n), C.byref(nb)), "rafting_log_gather")
    return refs[:n.value], blob, nb.value


def assert_same(got_refs, got_blob, want_refs, want_blob, where: str):
    assert len(got_refs) == len(want_refs), f"{where}: {len(got_refs)} refs, rafting_log_gather {len(want_refs)}"
    bad = np.flatnonzero(got_refs != want_refs)
    assert len(bad) == 0, f"{where}: ref {bad[0]} {got_refs[bad[0]]} != {want_refs[bad[0]]} ({len(bad)} differ)"
    for r in want_refs[(want_refs["len"] != ABSENT) & (want_refs["len"] > 0)]:
        o, n = int(r["blob_off"]), int(r["len"])
        assert np.array_equal(got_blob[o:o + n], want_blob[o:o + n]), f"{where}: payload of ({r['gid']}, {r['index']}) differs"


def check(e: engine.Engine, ranges, where: str, kind: str = "pageable", ticket: int = 0, slack: int = 0):
    """one gather under `ticket` held to rafting_log_gather -> (n_refs, bytes, host_served)"""
    g, f, c = arrays(ranges) if not isinstance(ranges, tuple) else ranges
    want_refs, want_blob, want_bytes = reference(e, g, f, c, 1 << 26)
    refs, blob = outputs(kind, int(c.sum()), want_bytes + slack)
    e.log_gather_begin(ticket, (g, f, c), refs, blob)
    n, nb, served = e.log_gather_wait(ticket)
    assert (n, nb) == (len(want_refs), want_bytes), where
    assert_same(refs[:n], blob, want_refs, want_blob, where)
    return n, nb, served


def payload(gid: int, index: int, term: int) -> bytes:
    """the payload bytes of an entry, a function of (gid, index, term); one in 11 is empty"""
    h = (gid * 2654435761 + index * 40503 + term * 97) & 0xFFFFFFFF
    n = 0 if h % 11 == 0 else 1 + h % 200
    return np.random.default_rng(h).integers(0, 256, n, dtype=np.uint8).tobytes()


def stored_engine(G: int, last_index: int, **log):
    cfg = abi.make_cfg(replicas=3, max_groups=G, max_rows=1, entry_pool_cap=64)
    e = engine.Engine(cfg)
    init = harness.init_array(G, terms=1)
    init["last_index"] = last_index
    init["last_term"] = 1
    e.open_bulk(0, init)
    if log is not None:
        e.log_config(**(log or dict(segment_bytes=1 << 20, hbm_segments=16, ring_slots=64)))
    return e


def random_ranges(rng, G: int, n: int, lo: int, hi: int, max_count: int):
    return [(int(rng.integers(0, G)), int(rng.integers(lo, hi)), int(rng.integers(0, max_count + 1))) for _ in range(n)]


def test_every_place_an_entry_lives(tmp_path):
    """A tiny arena over a pinned pool of 2 segments over an entry file, a ring of 16 slots, re-appended indices, indices
    never appended, zero-length payloads, and a FLUSH + rafting_log_trim: every output kind matches rafting_log_gather."""
    G = 48
    e = stored_engine(G, 400, segment_bytes=8192, hbm_segments=4, ring_slots=16)
    e.log_store_open(str(tmp_path / "entries.log"), cold_max_segments=2)
    rng = np.random.default_rng(3)
    for lo in range(1, 241, 40):
        batch = [(g, i, 1 + (i > 200), payload(g, i, 1 + (i > 200))) for g in range(G) for i in range(lo, lo + 40) if i % 17]
        rng.shuffle(batch)
        e.log_append(batch)
    e.log_append([(g, i, 2, payload(g, i, 2)) for g in range(0, G, 3) for i in range(230, 236)])   # re-appended at a newer term
    ib = abi.Inbox(1, G, 2)
    for g in range(0, G, 4):
        ib.flush(0, g, harness.T0, 30, 1)
    e.step(ib)
    dropped, _ = e.log_trim()
    assert dropped > 0
    served = 0
    for k, kind in enumerate(["pageable", "pinned", "misaligned"] * 2):
        ranges = random_ranges(rng, G, 160, -2, 260, 14) + [(5, 1, 40), (4, 20, 20), (9, 225, 16)]
        rng.shuffle(ranges)
        served += check(e, ranges, f"round {k} ({kind})", kind, ticket=k % 4)[2]
    st, fs = e.log_stats(), e.log_store_stats()
    assert served > 0 and st["hbm_hits"] > 0 and st["spilled_bytes"] > 0 and (st["cold_hits"] + fs["file_hits"]) > 0


def test_range_shapes():
    """count-0 ranges, overlapping and repeated ranges out of order, one range of 12 000 entries, 64 K ranges of 1-4 entries
    and an empty list"""
    G = 4096
    e = stored_engine(G, 20000, segment_bytes=1 << 22, hbm_segments=64, ring_slots=1 << 14)
    rng = np.random.default_rng(11)
    e.log_append([(7, i, 1, payload(7, i, 1)) for i in range(1, 12_101)])
    e.log_append([(g, i, 1, payload(g, i, 1)) for g in range(G) for i in range(1, 9)])
    check(e, [(3, 2, 0), (7, 5, 3), (7, 1, 0), (7, 4, 6), (7, 5, 3), (2, 8, 4), (1, 9, 0)], "count 0, overlapping, repeated")
    n, _, served = check(e, [(1, 1, 2), (7, 40, 12_000), (2, 3, 0)], "one long range", "pinned")
    assert n == 12_002 and served == 0
    g = rng.integers(0, G, 65536).astype(np.uint32)
    f = rng.integers(1, 8, 65536).astype(np.int64)
    c = rng.integers(1, 5, 65536).astype(np.uint32)
    n, _, _ = check(e, (g, f, c), "64 K short ranges", "pinned", ticket=3)
    assert n == int(c.sum())
    refs, blob = outputs("pageable", 0, 0)
    e.log_gather_begin(1, [], refs, blob)
    assert e.log_gather_wait(1) == (0, 0, 0)


def test_capacity():
    e = stored_engine(64, 400, segment_bytes=8192, hbm_segments=4, ring_slots=16)
    e.log_append([(g, i, 1, payload(g, i, 1)) for g in range(64) for i in range(1, 120)])
    ranges = [(g, 1 + 7 * g % 90, 25) for g in range(0, 64, 5)]
    g, f, c = arrays(ranges)
    want_refs, want_blob, need = reference(e, g, f, c, 1 << 24)
    n = int(c.sum())
    refs, blob = outputs("pageable", n, need)
    with pytest.raises(engine.RaftingError, match="E_CAPACITY"):             # refused at the begin, nothing enqueued
        e.log_gather_begin(0, ranges, refs, blob, refs_cap=n - 1)
    with pytest.raises(engine.RaftingError, match="E_INVAL"):                # the ticket is still free
        e.log_gather_wait(0)
    for kind in ("pageable", "pinned"):
        r2, b2 = outputs(kind, n, need + 64, fill=0xAB)
        e.log_gather_begin(0, ranges, r2, b2, blob_cap=need - 1)
        with pytest.raises(engine.RaftingError, match="E_CAPACITY") as ex:
            e.log_gather_wait(0)
        assert ex.value.sizes[1] == need, kind                               # the exact bytes
        assert (b2[need - 1:] == 0xAB).all(), kind                           # nothing past the cap
        e.log_gather_begin(0, ranges, r2, b2, blob_cap=ex.value.sizes[1])
        assert e.log_gather_wait(0)[:2] == (n, need)
        assert_same(r2[:n], b2, want_refs, want_blob, f"retry ({kind})")
        assert (b2[need:] == 0xAB).all()


def test_ordering_and_busy(tmp_path):
    e = stored_engine(256, 400)
    e.log_append([(g, i, 1, payload(g, i, 1)) for g in range(256) for i in range(1, 40)])
    refs, blob = outputs("pinned", 4096, 1 << 20)

    def batch(i):
        return [(g, i, 1, payload(g, i, 1)) for g in range(256)]

    def gathered(k):
        return e._gathered(refs[1024 * k:1024 * k + 256], blob[(1 << 18) * k:])

    # a begin right behind an append, with nothing synchronised in between, sees the appended entries
    e.log_append(batch(40))
    e.log_gather_begin(0, [(g, 40, 1) for g in range(256)], refs, blob)
    assert e.log_gather_wait(0)[0] == 256 and gathered(0) == batch(40)
    e.log_append(batch(41) + batch(42))
    for k in (1, 2):
        e.log_gather_begin(k, [(g, 40 + k, 1) for g in range(256)], refs[1024 * k:], blob[(1 << 18) * k:])
    busy = (lambda: e.log_append([(0, 99, 1, b"x")]), lambda: e.log_trim(), lambda: e.log_store_open(str(tmp_path / "f")))
    for call in busy:
        with pytest.raises(engine.RaftingError, match="E_BUSY"):
            call()
    assert e.log_gather_wait(1)[0] == 256
    for call in busy:                                                        # ticket 2 is still out
        with pytest.raises(engine.RaftingError, match="E_BUSY"):
            call()
    assert e.log_gather_wait(2) == (256, sum((len(p) + 15) & ~15 for *_, p in batch(42)), 0)
    assert gathered(1) == batch(41) and gathered(2) == batch(42)
    e.log_append([(0, 99, 1, b"x")])
    e.log_trim()


def test_two_tickets_and_a_step_gather_outstanding():
    G, rows = 1024, 2
    cfg = abi.make_cfg(replicas=3, max_groups=G, max_rows=rows)
    e = engine.Engine(cfg)
    e.open_bulk(0, harness.init_array(G, terms=np.arange(G) % 7))
    e.log_config(segment_bytes=1 << 20, hbm_segments=64, ring_slots=64)
    last = harness.elect_all(e, workload.make_wl(0x5EED0002, 1, G, 2))
    w = workload.make_wl(0x5EED0002, rows, G, 2)
    for k in range(2):
        ib = workload.leader_inbox_host(w, k, last)
        cout = compact.CompactOutbox(rows, G, 2, esc_cap=rows * G * 3)
        e.step_compact(compact.encode_inbox(ib, None, None, None), cout)
        last = compact.decode_outbox(cout)
        hi = cout.last_entry["x"]
        e.log_append([(g, i, int(cout.current_term[g]), payload(g, i, int(cout.current_term[g])))
                      for g in np.flatnonzero(hi > 0).tolist() for i in range(max(1, int(hi[g]) - 3), int(hi[g]) + 1)])
    want_step, _, _ = e.log_gather_step(0)
    rng = np.random.default_rng(5)
    sets = [random_ranges(rng, G, 300, 1, 12, 4) for _ in range(2)]
    wants = [reference(e, *arrays(s), 1 << 22) for s in sets]
    outs = [outputs(kind, int(arrays(s)[2].sum()), 1 << 22) for s, kind in zip(sets, ("pinned", "pageable"))]
    sr, sb, sp = np.zeros(1 << 16, e.ENTRY_REF), np.zeros(1 << 24, np.uint8), np.zeros(1 << 14, abi.PLAN_REF)
    e.log_gather_begin(2, sets[0], *outs[0])
    e.log_gather_step_begin(0, sr, sb, sp)
    e.log_gather_begin(3, sets[1], *outs[1])
    n_step = e.log_gather_step_wait(0)[0]
    for t, (r, b), (wr, wb, nb) in zip((3, 2), outs[::-1], wants[::-1]):
        assert e.log_gather_wait(t)[:2] == (len(wr), nb)
        assert_same(r[:len(wr)], b, wr, wb, f"ticket {t}")
    assert e._gathered(sr[:n_step], sb) == want_step


def test_misuse():
    e = stored_engine(64, 400)
    e.log_append([(1, i, 1, payload(1, i, 1)) for i in range(1, 10)])
    refs, blob = outputs("pageable", 64, 1 << 16)
    with pytest.raises(engine.RaftingError, match="E_INVAL"):
        e.log_gather_begin(4, [(1, 1, 3)], refs, blob)
    with pytest.raises(engine.RaftingError, match="E_INVAL"):
        e.log_gather_wait(0)
    with pytest.raises(engine.RaftingError, match="E_INVAL"):
        e.log_gather_begin(0, [(1, 1, 3), (64, 1, 1)], refs, blob)
    with pytest.raises(engine.RaftingError, match="E_INVAL"):                # a null blob with a non-zero cap
        engine._check(engine.lib().rafting_log_gather_begin(e._h, 0, 0, None, None, None, refs.ctypes.data, 64, None, 16), "begin")
    e.log_gather_begin(0, [(1, 1, 3)], refs, blob)
    with pytest.raises(engine.RaftingError, match="E_BUSY"):
        e.log_gather_begin(0, [(1, 1, 3)], refs, blob)
    assert e.log_gather_wait(0)[0] == 3
    cfg = abi.make_cfg(replicas=3, max_groups=64, max_rows=1)
    bare = engine.Engine(cfg)
    with pytest.raises(engine.RaftingError, match="E_INVAL"):                # no rafting_log_config
        bare.log_gather_begin(0, [(1, 1, 3)], refs, blob)
    # destroyed with a ticket outstanding: drained and freed (pinned outputs stay alive, the device may still be writing them)
    pr, pb = outputs("pinned", 64, 1 << 16)
    e.log_gather_begin(1, [(1, 1, 9)], pr, pb)
    e.close()
    assert pr["index"][:9].tolist() == list(range(1, 10))


# ---- the apply loop of a compact pump, pipelined ----

def with_submits(peers: tm.Peers, share: float = 0.05):
    """SUBMITs of 1..3 commands in the last row of a share of the groups of tests/timers_model's stream, so that its leaders
    replicate and commit entries"""
    inbox = peers.inbox

    def wrapped(k, planned, terms):
        ib = inbox(k, planned, terms)
        rng = np.random.default_rng(50_000 + k)
        r = ib.rows - 1
        for g in np.flatnonzero((rng.random(ib.n) < share) & (ib.op_meta[r] == 0)).tolist():
            ib.submit(r, g, peers.now(k), count=1 + g % 3)
        return ib
    peers.inbox = wrapped


class Applier:
    """The pump's apply side.  Per waited step: wait for the previous step's gather (appends are refused until then), append
    the payloads of the entries the step created, turn the step's commit records into apply ranges, begin their gather under
    the next ticket, and let it run while the next step does.  Every gather is held to rafting_log_gather; every applied
    entry's payload is payload(gid, index, term)."""

    def __init__(self, e: engine.Engine, G: int):
        self.e = e
        self.applied = np.zeros(G, np.int64)
        self.last = np.zeros(G, np.int64)
        self.commit = np.zeros(G, np.int64)
        self.seen = {}                                  # (gid, index) -> term of every applied entry
        self.out, self.k, self.entries = None, 0, 0

    def finish(self):
        if self.out is None:
            return
        ticket, refs, blob, want_refs, want_blob, nb, where = self.out
        assert self.e.log_gather_wait(ticket)[:2] == (len(want_refs), nb), where
        assert_same(refs[:len(want_refs)], blob, want_refs, want_blob, where)
        for (gid, index, term, data) in self.e._gathered(refs[:len(want_refs)], blob):
            assert data == payload(gid, index, term), f"{where}: ({gid}, {index}) applied bytes"
            self.seen[(gid, index)] = term
        self.entries += len(want_refs)
        self.out = None

    def on_wait(self, cout: compact.CompactOutbox, where: str):
        self.finish()
        gids = np.arange(cout.n) if cout.gids is None else cout.gids.astype(np.int64)
        hi = cout.last_entry["x"]
        ents = []
        for i in np.flatnonzero(hi > self.last[gids]).tolist():
            g, h = int(gids[i]), int(hi[i])
            t = int(cout.current_term[i])
            ents += [(g, x, t, payload(g, x, t)) for x in range(int(self.last[g]) + 1, h + 1)]
            self.last[g] = h
        if ents:
            self.e.log_append(ents)
        ob = abi.Outbox(1, cout.n, cout.F, cout.n)      # a compact outbox's group columns in a rafting_outbox_t
        ob.commit_index[:] = cout.commit_index
        ob.role_word[:] = cout.role_word
        ar = ingest.apply_ranges(ob, self.applied, None if cout.gids is None else cout.gids)
        self.commit[gids] = np.maximum(self.commit[gids], cout.commit_index)
        g, f = ar["gid"].astype(np.uint32), ar["first"].astype(np.int64)
        c = (ar["last"] - ar["first"] + 1).astype(np.uint32)
        want_refs, want_blob, nb = reference(self.e, g, f, c, 1 << 26)
        kind = ("pinned", "pageable")[self.k % 2]
        refs, blob = outputs(kind, int(c.sum()), nb)
        ticket = self.k % engine.Engine.GATHER_TICKETS
        self.e.log_gather_begin(ticket, (g, f, c), refs, blob)
        self.out = (ticket, refs, blob, want_refs, want_blob, nb, where)
        self.k += 1

    def close(self):
        self.finish()
        absent = [(g, i) for (g, i), t in self.seen.items() if t == 0]
        assert not absent, f"applied entries never appended: {absent[:4]}"
        for (g, i), t in sorted(self.seen.items())[::max(1, len(self.seen) // 3000)]:
            assert self.e.log_term(g, i) == t, (g, i)
        assert np.array_equal(self.applied, self.commit)


@pytest.mark.parametrize("flags", [0, abi.COMPACT_PREV_TERM])
def test_apply_loop_on_the_leader_stream(flags):
    """R = 3 leader stream, whole-shard and active compact steps alternating; each step's apply gather overlaps the next step"""
    G, R, rows = 4096, 3, 4
    cfg = abi.make_cfg(replicas=R, max_groups=G, max_rows=rows)
    ref, e = engine.Engine(cfg), engine.Engine(cfg)                        # ref: the dense run the stream's inboxes follow
    init = harness.init_array(G, terms=np.arange(G) % 7)
    ref.open_bulk(0, init)
    e.open_bulk(0, init)
    e.log_config(segment_bytes=1 << 22, hbm_segments=32, ring_slots=64)
    w1 = workload.make_wl(0x5EED0002, 1, G, R - 1)
    for sut in (ref, e):
        last = harness.elect_all(sut, w1)
    w = workload.make_wl(0x5EED0002, rows, G, R - 1)
    A = Applier(e, G)
    rng = np.random.default_rng(flags)
    for k in range(10):
        ib = workload.leader_inbox_host(w, k, last)
        last = ref.step(ib)
        gids = None if k % 2 == 0 else np.sort(rng.choice(G, G // 3, replace=False)).astype(np.uint32)
        ci = compact.encode_inbox(ib if gids is None else tm.slice_inbox(ib, gids), None, None, None)
        cout = compact.CompactOutbox(rows, G if gids is None else len(gids), R - 1, esc_cap=rows * G * R, gids=gids)
        e.step_compact(ci, cout, flags=flags)
        A.on_wait(cout, f"step {k}")
    A.close()
    assert A.entries > 10_000


@pytest.mark.parametrize("d", [0, 3])
def test_apply_loop_on_the_due_pump(d):
    """The 64 K x 3 due pump (host-listed and device-chosen tail positions) with SUBMITs, d steps in flight; every waited step's
    apply ranges are gathered under a ticket while the following steps run"""
    S = edit_pump.Stream(0)
    with_submits(S.P)
    pump = edit_pump.DuePump(S, d, "edit")
    pump.e.log_config(segment_bytes=1 << 22, hbm_segments=64, ring_slots=64)
    A = Applier(pump.e, edit_pump.G)
    tails = []

    def on_wait(j, cout):
        A.on_wait(cout, f"due tick {j}")
        tails.append(int(cout.counts[3]))

    pump.run(170, on_wait=on_wait)
    A.close()
    assert A.entries > 0 and max(tails) > 0


def test_natives_through_the_jni_glue(tmp_path):
    from tests import jni_exec
    from tests.jni_exec import Buf, buf_of_array, fn
    L = jni_exec.build(str(tmp_path))
    if L is None:
        pytest.skip("no gcc")
    e = stored_engine(64, 400)
    e.log_append([(g, i, 1, payload(g, i, 1)) for g in range(64) for i in range(1, 30)])
    g, f, c = arrays([(3, 2, 5), (9, 1, 0), (40, 20, 15), (5, 28, 4)])
    want_refs, want_blob, nb = reference(e, g, f, c, 1 << 20)
    L.fake_reset()
    begin = fn(L, "logGatherBegin", None, C.c_int64, C.c_int32, C.c_int32, C.POINTER(Buf), C.POINTER(Buf), C.POINTER(Buf),
               C.POINTER(Buf), C.c_int32, C.POINTER(Buf), C.c_int64)
    wait = fn(L, "logGatherWait", None, C.c_int64, C.c_int32, C.POINTER(jni_exec.Longs))
    refs, blob = np.zeros(len(want_refs), e.ENTRY_REF), np.zeros(1 << 16, np.uint8)
    h = e._h if isinstance(e._h, int) else e._h.value
    begin(h, 1, len(g), C.byref(buf_of_array(g)), C.byref(buf_of_array(f)), C.byref(buf_of_array(c)), C.byref(buf_of_array(refs)),
          len(refs), C.byref(buf_of_array(blob)), len(blob))
    res = np.zeros(3, np.int64)
    wait(h, 1, C.byref(jni_exec.Longs(3, res.ctypes.data_as(C.POINTER(C.c_int64)))))
    assert L.fake_throws() == 0, L.fake_thrown_message()
    assert res.tolist()[:2] == [len(want_refs), nb]
    assert_same(refs, blob, want_refs, want_blob, "jni")
    wait(h, 1, C.byref(jni_exec.Longs(3, res.ctypes.data_as(C.POINTER(C.c_int64)))))   # nothing in flight: RaftException
    assert L.fake_throws() == 1
