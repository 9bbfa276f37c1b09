"""tests/entry_model.py, the entry buffer's restatement, without a GPU: its visible reads against oracle/payload_model's
PayloadLog, its layout arithmetic against hand-worked examples, its index window against seglog.cuh's constant, and the
entry-buffer fuzz streams against the cases they exist to reach."""
import os

import numpy as np
import pytest

from oracle.payload_model import PayloadLog
from tests import entry_model as em

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def refs_of(entries, blob_off=None):
    """[(gid, index, term, payload)] -> (refs, blob), payloads packed back to back at their own offsets"""
    refs, blob = np.zeros(len(entries), em.ENTRY_REF), b""
    for k, (gid, index, term, p) in enumerate(entries):
        refs[k] = (gid, len(p), index, term, len(blob))
        blob += p
    return refs, blob


def test_window_constant_is_seglogs():
    with open(os.path.join(ROOT, "rafting_b200", "csrc", "seglog.cuh")) as f:
        assert em.window_constant(f.read()) == em.WINDOW


def test_reads_match_payload_log_without_window_events():
    rng = np.random.default_rng(4)
    m, p = em.EntryModel(8192, 4, 16), PayloadLog()
    for rnd in range(8):
        ents = [(0, int(i), 1 + rnd // 3, rng.bytes(int(rng.integers(0, 300)))) for i in rng.integers(1, 120, 90)]
        m.append(*refs_of(ents))
        for _, i, t, pay in ents:
            p.put(i, t, pay)
        for first in (1, 7, 50, 119):
            assert m.read(0, first, 40, 1 << 20, (1, 200, False))[0] == p.batch(first, 40)
    m.trim({0: (30, 200, False)}, 0, 1)
    p.flush(0, 30)
    for first in (1, 29, 30, 90):
        assert m.read(0, first, 200, 1 << 20, (30, 200, False))[0] == p.batch(first, 200)


def test_layout_tail_skip_exact_fit_and_sub_batch_split():
    S = 4096
    m = em.EntryModel(S, 3, 4)
    # 40 + 2000 -> 32 + 2000 = 2032 bytes; a second one needs 2032 more: 4064 <= 4096 fits; a third skips the 32-byte tail
    m.append(*refs_of([(0, 1, 1, b"a" * 2000), (0, 2, 1, b"b" * 2000), (0, 3, 1, b"c" * 2000)]))
    assert [m.find(0, i).off for i in (1, 2, 3)] == [0, 2032, 4096] and m.head == 4096 + 2032
    assert "tail skip" in m.seen
    # a record of S - 32 payload bytes fills a segment exactly: skip to 8192, end at 12288
    m.append(*refs_of([(0, 4, 1, b"d" * (S - 32))]))
    assert m.find(0, 4).off == 2 * S and m.head == 3 * S and "record fills a segment" in m.seen
    # a sub-batch ends within three segments of its head's segment: five whole-segment records go in sub-batches of 3 and 2
    m2 = em.EntryModel(S, 3, 4)
    m2.append(*refs_of([(1, i, 1, bytes([i]) * (S - 32)) for i in range(1, 6)]))
    assert [m2.find(1, i).off for i in range(1, 6)] == [0, S, 2 * S, 3 * S, 4 * S] and "sub-batch split" in m2.seen
    assert m2.stats["spilled_bytes"] == 2 * S and m2.resident(2 * S) and not m2.resident(S)
    # two segments: a whole-segment record after a partly filled segment starts at the boundary, in the same call
    m4 = em.EntryModel(S, 2, 4)
    m4.append(*refs_of([(3, 1, 1, b"a" * 100), (3, 2, 1, b"b" * (S - 32)), (3, 3, 1, b"c" * (S - 32))]))
    assert [m4.find(3, i).off for i in (1, 2, 3)] == [0, S, 2 * S] and m4.head == 3 * S
    # the ring's slot of index 1 with K = 4 also names 5: resident, but index 1 is served by the host
    m3 = em.EntryModel(S, 3, 4)
    m3.append(*refs_of([(2, 1, 1, b"x"), (2, 5, 1, b"y")]))
    assert not m3.served(2, 1) and m3.served(2, 5)


def test_window_rules():
    m = em.EntryModel(1 << 16, 4, 8)
    m.append(*refs_of([(0, i, 1, b"p") for i in range(1, 5)]))
    m.append(*refs_of([(0, 4 + em.WINDOW, 1, b"f")]))           # 4 + WINDOW < base + size + WINDOW = 5 + WINDOW: extends,
    g = m.groups[0]                                             # grows the window past WINDOW: cut to the newest WINDOW
    assert (g.base, g.size, sorted(g.entries)) == (5, em.WINDOW, [4 + em.WINDOW]) and "cut" in m.seen
    m.append(*refs_of([(0, 9 + 2 * em.WINDOW, 1, b"r")]))       # one past the window's end plus WINDOW: a new window
    assert (g.base, g.size) == (9 + 2 * em.WINDOW, 1) and "forward restart" in m.seen and m.stats["indexed"] == 1
    # one past a full window's end cuts its base away; a put of that base is then below the newest WINDOW indices: a new
    # window holding only it, not a window extended down and cut back past the index just put
    m = em.EntryModel(1 << 16, 4, 8)
    m.append(*refs_of([(0, 1, 1, b"a"), (0, 1 + em.WINDOW, 1, b"b"), (0, 1, 1, b"c")]))
    g = m.groups[0]
    assert (g.base, g.size, m.find(0, 1).payload, m.find(0, 1 + em.WINDOW)) == (1, 1, b"c", None) and m.stats["indexed"] == 1


@pytest.fixture(scope="module")
def streams():
    out = {}
    for case in em.CASES:
        s = em.Stream(case)
        for _ in s.ops():                                     # the same reads the GPU suite makes after every op
            s.m.gather(s.random_ranges(24), 0)
            s.m.gather(s.random_ranges(24), 0)
            s.m.gather(s.random_ranges(24), 0)
            rd, kv = s.reads()
            for gid, first, n, cap in rd:
                s.m.read(gid, first, n, cap, s.stored(gid))
            for gid, index in kv:
                s.m.export_kv(gid, index)
        out[case.name] = s.m.seen
    return out


@pytest.mark.parametrize("what", [
    "unaligned source", "shared source", "duplicate in a batch",
    "forward restart", "backward restart after a trim above the window", "restart below a full window", "restart below a trimmed empty window", "cut",
    "trim above the window", "ring slot holds a newer index",
    "tail skip", "sub-batch split", "spill skipped",
    "hbm read", "cold read", "file read",
    "index >= 2^32", "zero length", "record fills a segment",
])
def test_fuzz_streams_reach(streams, what):
    assert any(what in seen for seen in streams.values()), f"no entry-buffer fuzz stream reaches: {what}"
