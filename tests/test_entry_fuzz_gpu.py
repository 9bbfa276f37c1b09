"""The HBM entry buffer held to tests/entry_model.py, its plain restatement: seeded op streams (adversarial appends through
the raw C call, index-window restarts and cuts, FLUSH steps with trims, conflicting AppendEntries, close and reopen) with the
engine and the CPU oracle in lockstep, every read path checked against the model after each op; a compact leader stream
whose step gathers are held to the model; every blob cap around the need; and the two defects the model found."""
import ctypes as C

import numpy as np
import pytest

from oracle import binding
from rafting_b200 import abi, compact, engine, workload
from tests import entry_model as em
from tests import harness
from tests import timers_model as tm

pytestmark = pytest.mark.gpu

_PINNED = []
SENTINEL = 0xAB


def buffer(kind: str, nbytes: int, dtype=np.uint8) -> np.ndarray:
    """pageable, pinned, or pinned 8 bytes off a 16-byte boundary; every byte SENTINEL"""
    if kind == "pageable":
        a = np.full(max(nbytes, 16), SENTINEL, np.uint8)
    else:
        import torch
        skew = 8 if kind == "misaligned" else 0
        t = torch.full((max(nbytes, 16) + skew,), SENTINEL, dtype=torch.uint8, pin_memory=True)
        _PINNED.append(t)
        a = t.numpy()[skew:]
    return a[:nbytes].view(dtype) if nbytes else a[:0].view(dtype)


class Eng(engine.Engine):
    """the Engine plus the raw append the streams make, with the blob and refs as given"""
    entry_path = None

    def append_raw(self, refs: np.ndarray, blob: bytes):
        b = np.frombuffer(blob, np.uint8)
        engine._check(engine.lib().rafting_log_append(self._h, refs.ctypes.data, len(refs), b.ctypes.data, len(b)), "rafting_log_append")


def sync_gather(e, ranges, blob_cap: int, blob: np.ndarray | None = None):
    g, f, c = (np.array([r[k] for r in ranges], dt) for k, dt in enumerate((np.uint32, np.int64, np.uint32)))
    refs = np.zeros(max(int(c.sum()), 1), em.ENTRY_REF)
    blob = buffer("pageable", blob_cap + 64) if blob is None else blob
    n, nb = C.c_uint32(), C.c_size_t()
    rc = engine.lib().rafting_log_gather(e._h, len(g), g.ctypes.data, f.ctypes.data, c.ctypes.data, refs.ctypes.data, len(refs),
                                         blob.ctypes.data, blob_cap, C.byref(n), C.byref(nb))
    return rc, refs[:n.value], blob, nb.value


def assert_refs(got, blob, want, pays, where):
    assert len(got) == len(want), f"{where}: {len(got)} refs, model {len(want)}"
    bad = np.flatnonzero(got != want)
    assert len(bad) == 0, f"{where}: ref {bad[0]} {got[bad[0]]} != model {want[bad[0]]} ({len(bad)} differ)"
    for k, r in enumerate(want):
        if pays[k]:
            o = int(r["blob_off"])
            assert blob[o:o + len(pays[k])].tobytes() == pays[k], f"{where}: payload of ({r['gid']}, {r['index']}) differs"


def check_all(e, s: em.Stream, where: str, k: int):
    m = s.m
    # sync gather into exactly the bytes the model needs
    ranges = s.random_ranges(24)
    want, pays, need, host, _ = m.gather(ranges, 0)
    rc, got, blob, nb = sync_gather(e, ranges, need)
    assert rc == 0 and nb == need, f"{where}: rafting_log_gather rc {rc}, {nb} bytes, model {need}"
    assert_refs(got, blob, want, pays, f"{where} sync")
    assert (blob[need:] == SENTINEL).all(), f"{where}: sync gather wrote past the need"
    # two range gathers outstanding at once, into two output kinds
    kinds = ["pageable", "pinned", "misaligned"]
    plans = []
    for t in range(2):
        rs = s.random_ranges(24)
        w = m.gather(rs, 0)
        refs, b = buffer(kinds[(k + t) % 3], 32 * max(len(w[0]), 1), em.ENTRY_REF), buffer(kinds[(k + t + 1) % 3], w[2] + 32)
        e.log_gather_begin(t, rs, refs, b, refs_cap=len(w[0]), blob_cap=w[2])
        plans.append((w, refs, b))
    for t, ((want, pays, need, host, _), refs, b) in enumerate(plans):
        n, nb, served = e.log_gather_wait(t)
        assert (n, nb, served) == (len(want), need, host), f"{where} ticket {t}: {(n, nb, served)} != model {(len(want), need, host)}"
        assert_refs(refs[:n], b, want, pays, f"{where} ticket {t}")
        assert (b[need:need + 32] == SENTINEL).all()
    # visible reads, and the tier each payload came from
    rd, kv = s.reads()
    for gid, first, max_n, cap in rd:
        before = {**e.log_stats(), **e.log_store_stats()} if s.case.entry_file else e.log_stats()
        want, tiers = m.read(gid, first, max_n, cap, s.stored(gid))
        assert e.log_read(gid, first, max_n, blob_cap=cap) == want, f"{where}: log_read({gid}, {first}, {max_n}, {cap})"
        after = {**e.log_stats(), **e.log_store_stats()} if s.case.entry_file else e.log_stats()
        for t, key in (("hbm", "hbm_hits"), ("cold", "cold_hits"), ("file", "file_hits")):
            if key in after:
                assert after[key] - before[key] == tiers.count(t), f"{where}: log_read({gid}, {first}) {key}"
    for gid, index in kv:
        want = m.export_kv(gid, index)
        if want is None:
            with pytest.raises(engine.RaftingError, match="E_INVAL"):
                e.log_export_kv(gid, index, cap=1 << 17)
        else:
            assert e.log_export_kv(gid, index, cap=1 << 17) == want, f"{where}: export_kv({gid}, {index})"
    st = e.log_stats()
    assert {k: st[k] for k in m.stats} == m.stats, f"{where}: stats {st} != model {m.stats}"


@pytest.mark.parametrize("case", em.CASES, ids=lambda c: c.name)
def test_op_stream(case, tmp_path):
    e = Eng(abi.make_cfg(replicas=3, max_groups=case.G, max_rows=1, entry_pool_cap=64))
    e.entry_path = str(tmp_path / "entries.log")
    s = em.Stream(case, eng=e)
    for k, label in enumerate(s.ops()):
        where = f"{case.name} op {k} ({label})"
        for gid in range(0, case.G, 7):
            a, b = s.o.export(gid), e.export(gid)
            assert (a.first_index, a.last_index, a.term_runs) == (b.first_index, b.last_index, b.term_runs), where
        check_all(e, s, where, k)


# ---- step gathers ------------------------------------------------------------------------------------------------------
def step_stream(steps: int, on_step):
    """the R = 3 leader stream over 512 groups, stepped by the oracle and, as compact steps (whole shard, then active), by
    the engine under test; on_step(k, e, o, m, rng, cout, gids) after each engine step"""
    G, R, rows, seed = 512, 3, 4, 0x5EED0002
    cfg = abi.make_cfg(replicas=R, max_groups=G, max_rows=rows)
    o, e = binding.Oracle(cfg), Eng(cfg)
    init = harness.init_array(G, terms=np.arange(G) % 7)
    o.open_bulk(0, init)
    e.open_bulk(0, init)
    log = dict(segment_bytes=16384, hbm_segments=4, ring_slots=4)
    e.log_config(**log)
    w1 = workload.make_wl(seed, 1, G, R - 1)
    last = harness.elect_all(o, w1)
    harness.elect_all(e, w1)
    w = workload.make_wl(seed, rows, G, R - 1)
    rng = np.random.default_rng(seed)
    m = em.EntryModel(log["segment_bytes"], log["hbm_segments"], log["ring_slots"])
    for k in range(steps):
        ib = workload.leader_inbox_host(w, k, last)
        last = o.step(ib)
        gids = None if k % 2 == 0 else np.sort(rng.choice(G, G // 3, replace=False)).astype(np.uint32)
        ci = compact.encode_inbox(ib if gids is None else tm.slice_inbox(ib, gids), None, None, None)
        cout = compact.CompactOutbox(rows, G if gids is None else len(gids), R - 1, esc_cap=rows * G * R, gids=gids)
        e.step_compact(ci, cout)
        on_step(k, e, o, m, rng, cout, gids)


def append_created(e, m, rng, cout, gids, k):
    """the created entries with adversarial payloads and duplicates; some groups' windows restart forward past them, and the
    next step's append takes those groups back (a backward restart)"""
    g = np.arange(cout.n) if gids is None else np.asarray(gids, np.int64)
    hi = cout.last_entry["x"]
    ents = []
    for i in np.flatnonzero(hi > 0):
        gid, h = int(g[i]), int(hi[i])
        ents += [(gid, x, int(cout.current_term[i]), em.payload_len(rng, 16384) // 4) for x in range(max(1, h - 6), h + 1)]
        r = rng.random()
        if r < 0.03:
            ents.append((gid, h + 2 * em.WINDOW, 1, 40))                         # forward restart: the created ones drop out
        elif r < 0.06:
            ents.append((gid, h + (1 << 32), 1, 24))                              # same low 32 bits, same ring slot
    if ents:
        ents += [ents[int(j)][:3] + (int(rng.integers(0, 90)),) for j in rng.integers(0, len(ents), len(ents) // 20)]
        ents = [ents[j] for j in rng.permutation(len(ents))]
        refs, blob = em.adversarial_batch(rng, ents, 16384)
        m.append(refs, blob)
        e.append_raw(refs, blob)


def flush_and_trim(o, e, m, rng):
    """FLUSH a few entries off the front of up to 64 groups' logs on both sides, then rafting_log_trim of each such group with
    the stored range the oracle exports: their index floors go up under the entries the next steps gather.  Only groups whose
    stored range the engine's active steps left equal to the oracle's are flushed."""
    G = e.G
    ib = abi.Inbox(1, G, 2)
    flushed = []
    for gid in rng.choice(G, 64, replace=False).tolist():
        a, b = o.export(gid), e.export(gid)
        lo, hi = int(a.first_index), int(a.last_index)
        if int(a.term_runs) and hi - lo >= 2 and (a.first_index, a.last_index, a.term_runs) == (b.first_index, b.last_index, b.term_runs):
            x = lo + int(rng.integers(1, min(hi - lo, 4) + 1))
            ib.flush(0, gid, harness.T0, x, o.log_term(gid, x))
            flushed.append(gid)
    o.step(ib)
    e.step(ib)
    dropped = 0
    for gid in flushed:
        a, b = o.export(gid), e.export(gid)
        assert (a.first_index, a.last_index, a.term_runs) == (b.first_index, b.last_index, b.term_runs), gid
        want = m.trim({gid: (int(a.first_index), int(a.last_index), int(a.term_runs) == 0)}, gid, 1)
        assert e.log_trim(gid, 1) == want, gid
        dropped += want[0]
    assert dropped > 0


def check_step(e, m, cout, gids, where, kinds=("pageable", "pinned", "misaligned")):
    t, g, f, c = em.dense_ranges(e, 0, cout.rows, cout.n, gids)
    want, pays, need, host, plans = m.gather_step(t, g, f, c)
    for kind in kinds:
        refs, blob = buffer(kind, 32 * max(len(want), 1), em.ENTRY_REF), buffer(kind, need + 32)
        pl = buffer(kind, 16 * max(len(t), 1), abi.PLAN_REF)
        e.log_gather_step_begin(0, refs, blob, pl, refs_cap=len(want), blob_cap=need, plans_cap=len(t))
        n, nb, npl, served = e.log_gather_step_wait(0)
        assert (n, nb, npl, served) == (len(want), need, len(t), host), f"{where} ({kind}): {(n, nb, npl, served)} != model"
        assert_refs(refs[:n], blob, want, pays, f"{where} ({kind})")
        assert np.array_equal(pl[:npl], plans), f"{where} ({kind}): plan records"
        assert (blob[need:need + 32] == SENTINEL).all()
    return len(want), host


def test_step_gathers_with_restarts_and_duplicates():
    seen = {"refs": 0, "host": 0}

    def on_step(k, e, o, m, rng, cout, gids):
        append_created(e, m, rng, cout, gids, k)
        n, h = check_step(e, m, cout, gids, f"step {k} ({'whole' if gids is None else 'active'})")
        seen["refs"] += n
        seen["host"] += h
        if k % 3 == 1:
            flush_and_trim(o, e, m, rng)
    step_stream(9, on_step)
    assert seen["refs"] > 0 and 0 < seen["host"] < seen["refs"]


def test_every_blob_cap_around_the_need():
    """for caps need - 16 ... need, the sync, range and step gathers decide alike, report the need, and leave every byte past
    the cap alone: over a step's plan ranges (all three gathers) and over random ranges (sync and range gathers)"""
    done = []

    def on_step(k, e, o, m, rng, cout, gids):
        append_created(e, m, rng, cout, gids, k)
        if k == 2:
            flush_and_trim(o, e, m, rng)
        if k < 3:
            return
        t, g, f, c = em.dense_ranges(e, 0, cout.rows, cout.n, gids)
        sweep(e, m, list(zip(g.tolist(), f.tolist(), c.tolist())), t)
        held = [gid for gid, grp in m.groups.items() if grp.entries]
        for _ in range(3):
            ranges = []
            for gid in rng.choice(held, 40).tolist():
                i = sorted(m.groups[gid].entries)[int(rng.integers(0, len(m.groups[gid].entries)))]
                ranges.append((gid, max(1, i - int(rng.integers(0, 4))), int(rng.integers(0, 13))))
            sweep(e, m, ranges, None)
        done.append(k)
    step_stream(5, on_step)
    assert done


def sweep(e, m, ranges, t):
    """every cap from need - 16 to need over ranges; t: the step's plan lane slots when ranges are its plans, else None"""
    n = sum(r[2] for r in ranges)
    _, _, need, _, _ = m.gather(ranges, 0)
    assert need > 16
    for cap in range(need - 16, need + 1):
        fits = need <= cap
        rc, _, blob, nb = sync_gather(e, ranges, cap)
        assert (rc == 0) == fits and (not fits or nb == need), f"cap {cap}: sync rc {rc}, {nb} bytes, need {need}"
        assert (blob[cap:] == SENTINEL).all(), f"cap {cap}: the sync gather wrote past the cap"
        refs, b = buffer("pinned", 32 * n, em.ENTRY_REF), buffer("pageable", cap + 64)
        e.log_gather_begin(1, ranges, refs, b, blob_cap=cap)
        if fits:
            assert e.log_gather_wait(1)[1] == need
        else:
            with pytest.raises(engine.RaftingError, match="E_CAPACITY") as ex:
                e.log_gather_wait(1)
            assert ex.value.sizes[1] == need
        assert (b[cap:] == SENTINEL).all(), f"cap {cap}: the range gather wrote past the cap"
        if t is None:
            continue
        refs, b, pl = np.zeros(n, em.ENTRY_REF), buffer("pinned", cap + 64), np.zeros(len(t), abi.PLAN_REF)
        e.log_gather_step_begin(0, refs, b, pl, blob_cap=cap)
        if fits:
            assert e.log_gather_step_wait(0)[1] == need
        else:
            with pytest.raises(engine.RaftingError, match="E_CAPACITY") as ex:
                e.log_gather_step_wait(0)
            assert ex.value.sizes[1] == need
        assert (b[cap:] == SENTINEL).all(), f"cap {cap}: the step gather wrote past the cap"


# ---- the defects the model found -----------------------------------------------------------------------------------------------
def test_sync_gather_never_writes_past_blob_cap():
    """one resident entry of one byte and a one-byte cap: the aligned need is 16, so rafting_log_gather refuses, as the range
    gather does, instead of copying 16 bytes into the caller's one"""
    e = Eng(abi.make_cfg(replicas=3, max_groups=4, max_rows=1))
    e.log_config(segment_bytes=4096, hbm_segments=4, ring_slots=4)
    e.log_append([(0, 1, 1, b"x")])
    rc, _, blob, _ = sync_gather(e, [(0, 1, 1)], 1)
    assert rc == -5 and (blob[1:] == SENTINEL).all()
    refs, b = np.zeros(1, em.ENTRY_REF), buffer("pageable", 64)
    e.log_gather_begin(0, [(0, 1, 1)], refs, b, blob_cap=1)
    with pytest.raises(engine.RaftingError, match="E_CAPACITY"):
        e.log_gather_wait(0)
    rc, refs, blob, nb = sync_gather(e, [(0, 1, 1)], 16)
    assert rc == 0 and nb == 16 and blob[0] == ord("x")


@pytest.mark.parametrize("emptied", [False, True], ids=["window above", "window trimmed empty"])
def test_restart_below_a_trimmed_window_is_served_from_hbm(emptied):
    """a group whose log was trimmed above WINDOW + 1 is closed and reopened for a context that starts again at index 1: its
    new entries are resident and the ring holds them, so the device serves every one (none is left to the host)"""
    G, H = 4, em.HIGH
    cfg = abi.make_cfg(replicas=3, max_groups=G, max_rows=1, entry_pool_cap=8)
    e = Eng(cfg)
    init = harness.init_array(G, terms=1)
    init["epoch_index"], init["epoch_term"], init["commit_index"] = H, 1, H
    init["first_index"], init["last_index"], init["last_term"] = H + 1, H + 100, 1
    e.open_bulk(0, init)
    e.log_config(segment_bytes=1 << 16, hbm_segments=8, ring_slots=64)
    e.log_append([(1, H + i, 1, b"old %d" % i) for i in range(1, 51)])
    ib = abi.Inbox(1, G, 2)
    ib.flush(0, 1, harness.T0, H + (80 if emptied else 40), 1)
    e.step(ib)
    assert e.log_trim()[0] == (50 if emptied else 39)
    e.close_group(1)
    e.open_group(1, term=1, last_index=50, last_term=1)
    new = [(1, i, 1, b"new %d" % i) for i in range(1, 51)]
    e.log_append(new)
    refs, b = np.zeros(50, em.ENTRY_REF), buffer("pageable", 50 * 16)
    e.log_gather_begin(0, [(1, 1, 50)], refs, b)
    n, nb, served = e.log_gather_wait(0)
    assert e._gathered(refs[:n], b) == [(g, i, t, p) for g, i, t, p in new]
    assert served == 0, f"{served} of 50 resident entries served by the host"


def test_put_below_a_full_window_starts_a_new_window():
    """(g, 1), (g, 2^22 + 1), (g, 1) in one append: the second put grows the window past WINDOW and cuts index 1 away, so the
    third is below the newest WINDOW indices and starts a new window holding only it (extending the window down to it and
    cutting back would drop the very index being put)"""
    e = Eng(abi.make_cfg(replicas=3, max_groups=4, max_rows=1))
    e.log_config(segment_bytes=4096, hbm_segments=4, ring_slots=4)
    e.log_append([(2, 1, 1, b"first"), (2, 1 + em.WINDOW, 1, b"far"), (2, 1, 3, b"again")])
    assert e.log_stats()["indexed"] == 1
    assert e.log_gather([(2, 1, 1), (2, 1 + em.WINDOW, 1)]) == [(2, 1, 3, b"again"), (2, 1 + em.WINDOW, 0, None)]
    refs, b = np.zeros(2, em.ENTRY_REF), buffer("pageable", 64)
    e.log_gather_begin(0, [(2, 1, 2)], refs, b)
    assert e.log_gather_wait(0) == (2, 16, 1)                    # index 2 was never put; index 1 is served by the device
    e.log_append([(2, 2, 3, b"next")])
    assert e.log_gather([(2, 1, 2)]) == [(2, 1, 3, b"again"), (2, 2, 3, b"next")]


def test_two_segment_arena_takes_whole_segment_records():
    """hbm_segments = 2: a record that fills a segment, after a partly filled one, starts at the boundary instead of failing
    the append, in the same call and in the next"""
    e = Eng(abi.make_cfg(replicas=3, max_groups=4, max_rows=1))
    e.log_config(segment_bytes=4096, hbm_segments=2, ring_slots=4)
    big = [bytes([i]) * (4096 - 32) for i in range(4)]
    e.log_append([(0, 1, 1, b"a" * 100), (0, 2, 1, big[0]), (0, 3, 1, big[1])])
    e.log_append([(0, 4, 1, b"b" * 7), (0, 5, 1, big[2])])
    assert e.log_stats()["head"] == 5 * 4096
    assert e.log_gather([(0, 1, 5)]) == [(0, 1, 1, b"a" * 100), (0, 2, 1, big[0]), (0, 3, 1, big[1]), (0, 4, 1, b"b" * 7),
                                         (0, 5, 1, big[2])]
